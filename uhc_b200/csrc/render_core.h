// render_core.h -- the offline renderer's per-frame and per-pixel arithmetic (include/uhc_render.h), for the device (render.cu) and, with
// -DUHC_EMU, for the host emulation the CPU tests run (tests/emu/render_emu.cpp).
//
// The pixel path uses only fp32 + - * / and sqrt (plus floorf, which is exact), so a device build without contracted multiply-adds
// (render.cu: -fmad=false, IEEE division and square root) and a host build with -ffp-contract=off give the same bits.  The camera basis is
// built on the host in fp64 (camera_setup) and handed over in fp32: no trigonometric function runs per pixel.
//
// shade_pixel is templated on the scene: the hulls (Scene, cast below) or the skinned mesh (render_mesh_core.h's MeshScene and its cast), so
// both renderers share the camera, floor, checker, colours, shading and to_u8.
//
// A pose table row holds, per body, R (row-major 3x3, body -> world) and the body origin p: world = R v + p.  Hull planes are in body
// frame, n . v + d <= 0 inside.
#pragma once
#include <math.h>
#include "motion_core.h"

#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_RDEV __device__ __forceinline__
#else
#define UHC_RDEV static inline
#endif

namespace uhc {
namespace render {

constexpr int NB = 24, POSE = 12;
constexpr int LABEL_SKY = 0, LABEL_FLOOR = 1, LABEL_BODY = 2;        // body b of humanoid h: LABEL_BODY + 24 h + b
// one directional light (unit vector towards it), ambient + Lambert weights, colours (linear, 0..1)
constexpr float LIGHT_X = 0.26726124f, LIGHT_Y = -0.53452248f, LIGHT_Z = 0.80178373f;    // (1, -2, 3) / sqrt(14)
constexpr float AMBIENT = 0.35f, DIFFUSE = 0.65f;
constexpr float SKY_R = 0.62f, SKY_G = 0.74f, SKY_B = 0.86f;
constexpr float FLOOR0 = 0.60f, FLOOR1 = 0.42f;                      // the two squares of the checker (grey), 1 m wide
constexpr float CHECK = 1.0f, FLOOR_FAR = 60.0f;                     // floor hits farther than FLOOR_FAR (m) are sky
constexpr float HUMANOID_R = 0.70f, HUMANOID_G = 0.70f, HUMANOID_B = 0.70f;   // the humanoid grey
constexpr float GHOST_R = 0.70f, GHOST_G = 0.0f, GHOST_B = 0.0f;              // the ghost red (eval_relive.py's geom_rgba)
constexpr float SHADOW_EPS = 1e-4f;                                  // a shadow ray starts this far (m) from its surface point
constexpr float INF = __builtin_huge_valf();

// the camera as the pixel path reads it: eye = look + off; ray of pixel (x, y) = fwd + a right + b up, a = 2 (x + 0.5) / W - 1,
// b = 1 - 2 (y + 0.5) / H, right / up pre-scaled by tan(fovy / 2) (right also by W / H)
struct Cam {
    float look[3], off[3], fwd[3], right[3], up[3];
    float shift;                 // ghost x offset
    int focus, visible;          // visible: bit h = humanoid h is drawn
};

// the scene of one frame: the variant's planes, every body's pose and world bounding sphere (slot j = 24 h + b)
struct Scene {
    const float *plane;          // [nplane][4] of the frame's variant
    const int *adr, *num;        // [24]
    const float *pose;           // [48][POSE]
    const float *sph;            // [48][4]: world centre, radius
    int visible;
};

#ifdef UHC_RENDER_HOST
// host only: MuJoCo's free camera (mjv_cameraInModel: forward = (ce ca, ce sa, se), up = (-se ca, -se sa, ce)) in fp64, rounded once
template <class CamIn>
inline void camera_setup(const CamIn &c, int W, int H, int humanoids, Cam *out) {
    const double pi = 3.14159265358979323846, az = c.azimuth * pi / 180, el = c.elevation * pi / 180;
    const double ca = cos(az), sa = sin(az), ce = cos(el), se = sin(el), th = tan(c.fovy * pi / 360);
    const double f[3] = {ce * ca, ce * sa, se}, u[3] = {-se * ca, -se * sa, ce}, r[3] = {sa, -ca, 0.0};
    const double asp = (double)W / (double)H;
    for (int k = 0; k < 3; k++) {
        out->look[k] = (float)c.lookat[k];
        out->off[k] = (float)(-c.distance * f[k]);
        out->fwd[k] = (float)f[k];
        out->right[k] = (float)(r[k] * th * asp);
        out->up[k] = (float)(u[k] * th);
    }
    out->shift = (float)c.shift_expert;
    out->focus = c.focus != 0;
    out->visible = (c.hide_im ? 0 : 1) | ((humanoids > 1 && !c.hide_expert) ? 2 : 0);
}

// host only: the argument checks every trace shares (nullptr: none fails)
template <class CamIn>
inline const char *frame_args_error(const CamIn *c, int W, int H, long n) {
    if (!c) return "null camera";
    if (n < 0) return "n < 0";
    if (W < 1 || H < 1 || W > 16384 || H > 16384) return "W and H must be in 1 .. 16384";
    const double v[8] = {c->lookat[0], c->lookat[1], c->lookat[2], c->azimuth, c->elevation, c->distance, c->fovy, c->shift_expert};
    for (double x : v) if (!isfinite(x)) return "camera needs finite values, distance > 0 and 0 < fovy < 180";
    if (!(c->distance > 0) || !(c->fovy > 0 && c->fovy < 180)) return "camera needs finite values, distance > 0 and 0 < fovy < 180";
    return nullptr;
}
#endif

// ---- the pose pass (fp64): body world positions / quaternions of one qpos (motion_core.h's FK with the frame's variant table `body`)
UHC_RDEV void pose_fk(const motion::MotionModel &m, const double *q, const double *body, double *wpos, double *wq) {
    double bq[4 * motion::MB];
    motion::m_local_quats(q, bq);
    for (int b = 0; b < motion::MB; b++) motion::m_fk_body(m, b, q, bq, body, wpos, wq);
}
// -> pose rows [24][POSE]: R of the normalised quaternion (motion_lib.qmat), then the position
template <class Out>
UHC_RDEV void pose_rows(const double *wpos, const double *wq, Out *out) {
    for (int b = 0; b < NB; b++) {
        const double *c = wq + 4 * b;
        const double nrm = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2] + c[3] * c[3]);
        const double w = c[0] / nrm, x = c[1] / nrm, y = c[2] / nrm, z = c[3] / nrm;
        const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                             2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                             2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
        Out *o = out + POSE * b;
        for (int k = 0; k < 9; k++) o[k] = (Out)R[k];
        for (int k = 0; k < 3; k++) o[9 + k] = (Out)wpos[3 * b + k];
    }
}

// ---- the pixel path (fp32)
UHC_RDEV float dot3(const float *a, const float *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// staging of body slot j of a frame: its pose (the ghost shifted by cam.shift in x) and the world sphere of its hull
UHC_RDEV void stage_body(const float *src, const float *sphere_body, int ghost, float shift, float *pose, float *sph) {
    for (int k = 0; k < POSE; k++) pose[k] = src[k];
    if (ghost) pose[9] = pose[9] + shift;
    const float *c = sphere_body;
    for (int i = 0; i < 3; i++) sph[i] = ((pose[3 * i] * c[0] + pose[3 * i + 1] * c[1]) + pose[3 * i + 2] * c[2]) + pose[9 + i];
    sph[3] = c[3];
}

// Cyrus-Beck clip of the body-frame ray o + t d, t in [t0, t1], against `num` planes: -2 = miss, else the entering plane (-1: the ray
// starts inside at t0) with *tin = the entering distance
UHC_RDEV int clip_hull(const float *pl, int num, const float *o, const float *d, float t0, float t1, float *tin) {
    int kin = -1;
    for (int k = 0; k < num; k++) {
        const float *p = pl + 4 * k;
        const float den = dot3(p, d);
        const float nu = -(dot3(p, o) + p[3]);
        if (den < 0.0f) { const float t = nu / den; if (t > t0) { t0 = t; kin = k; } }
        else if (den > 0.0f) { const float t = nu / den; if (t < t1) t1 = t; }
        else if (nu < 0.0f) return -2;
        if (t0 > t1) return -2;
    }
    *tin = t0;
    return kin;
}

// the ray o + t d (world, |d| = 1) against every visible body, t in (t_lo, *t_best): the nearest hit's slot (-1: none), *t_best and its
// world normal nw updated.  any: stop at the first hit (shadow rays).
UHC_RDEV int cast(const Scene &s, const float *o, const float *d, float t_lo, float *t_best, float *nw, bool any) {
    int hit = -1, hk = -1;
    for (int h = 0; h < 2; h++) {
        if (!((s.visible >> h) & 1)) continue;
        for (int b = 0; b < NB; b++) {
            const int j = h * NB + b;
            const float *sp = s.sph + 4 * j;
            const float oc[3] = {sp[0] - o[0], sp[1] - o[1], sp[2] - o[2]};
            // squared distance of the centre from the ray through its perpendicular (no cancellation of two squares of the eye distance)
            const float bp = dot3(oc, d), r2 = sp[3] * sp[3];
            const float q[3] = {oc[0] - bp * d[0], oc[1] - bp * d[1], oc[2] - bp * d[2]};
            const float disc = r2 - dot3(q, q);
            if (disc < 0.0f) continue;
            const bool outside = dot3(oc, oc) > r2;
            if (outside && (bp < 0.0f || bp - sqrtf(disc) >= *t_best)) continue;   // behind the origin, or beyond the nearest hit
            const float *P = s.pose + POSE * j;
            const float w[3] = {o[0] - P[9], o[1] - P[10], o[2] - P[11]};
            float ob[3], db[3];
            for (int k = 0; k < 3; k++) {
                ob[k] = (P[k] * w[0] + P[3 + k] * w[1]) + P[6 + k] * w[2];
                db[k] = (P[k] * d[0] + P[3 + k] * d[1]) + P[6 + k] * d[2];
            }
            float tin;
            const int k = clip_hull(s.plane + 4 * s.adr[b], s.num[b], ob, db, t_lo, *t_best, &tin);
            if (k == -2 || !(tin < *t_best)) continue;
            *t_best = tin; hit = j; hk = k;
            if (any) return hit;
        }
    }
    if (hit >= 0) {
        if (hk >= 0) {
            const float *n = s.plane + 4 * (s.adr[hit % NB] + hk), *P = s.pose + POSE * hit;
            for (int i = 0; i < 3; i++) nw[i] = (P[3 * i] * n[0] + P[3 * i + 1] * n[1]) + P[3 * i + 2] * n[2];
        } else { nw[0] = -d[0]; nw[1] = -d[1]; nw[2] = -d[2]; }
    }
    return hit;
}

UHC_RDEV unsigned char to_u8(float c) { return (unsigned char)((c > 1.0f ? 1.0f : (c < 0.0f ? 0.0f : c)) * 255.0f + 0.5f); }

// the first humanoid's root x, y (before any shift), where a focused camera looks
UHC_RDEV void focus_xy(const Scene &s, float *look) { look[0] = s.pose[9]; look[1] = s.pose[10]; }

// pixel (x, y) of a W x H frame: rgb, depth (+inf on sky), label.  S is the frame's scene: Scene (the hulls) or, through the overloads of
// cast and focus_xy that render_mesh_core.h adds, MeshScene (the skinned mesh); camera, floor, checker, colours and shading are shared.
template <class S>
UHC_RDEV void shade_pixel(const Cam &cam, const S &s, int x, int y, int W, int H, unsigned char *rgb, float *depth, unsigned char *label) {
    float look[3] = {cam.look[0], cam.look[1], cam.look[2]};
    if (cam.focus) focus_xy(s, look);
    const float o[3] = {look[0] + cam.off[0], look[1] + cam.off[1], look[2] + cam.off[2]};
    const float a = 2.0f * ((float)x + 0.5f) / (float)W - 1.0f, b = 1.0f - 2.0f * ((float)y + 0.5f) / (float)H;
    float d[3];
    for (int k = 0; k < 3; k++) d[k] = (cam.fwd[k] + a * cam.right[k]) + b * cam.up[k];
    const float inv = 1.0f / sqrtf(dot3(d, d));
    for (int k = 0; k < 3; k++) d[k] = d[k] * inv;
    float t = INF, nw[3] = {0.0f, 0.0f, 1.0f};
    int lab = LABEL_SKY;
    if (d[2] < 0.0f) {
        const float tf = -o[2] / d[2];
        if (tf > 0.0f && tf < FLOOR_FAR) { t = tf; lab = LABEL_FLOOR; }
    }
    const int j = cast(s, o, d, 0.0f, &t, nw, false);
    if (j >= 0) lab = LABEL_BODY + j;
    float c[3] = {SKY_R, SKY_G, SKY_B};
    if (lab != LABEL_SKY) {
        const float p[3] = {o[0] + t * d[0], o[1] + t * d[1], o[2] + t * d[2]};
        float base[3];
        if (lab == LABEL_FLOOR) {
            const float sq = floorf(p[0] / CHECK) + floorf(p[1] / CHECK);
            const float g = (sq - 2.0f * floorf(sq * 0.5f)) == 0.0f ? FLOOR0 : FLOOR1;
            base[0] = g; base[1] = g; base[2] = g;
        } else if (j < NB) {
            base[0] = HUMANOID_R; base[1] = HUMANOID_G; base[2] = HUMANOID_B;
        } else {
            base[0] = GHOST_R; base[1] = GHOST_G; base[2] = GHOST_B;
        }
        const float L[3] = {LIGHT_X, LIGHT_Y, LIGHT_Z};
        float ndl = dot3(nw, L);
        if (ndl > 0.0f) {
            float ts = INF, ns[3];
            if (cast(s, p, L, SHADOW_EPS, &ts, ns, true) >= 0) ndl = 0.0f;
        } else ndl = 0.0f;
        const float k = AMBIENT + DIFFUSE * ndl;
        for (int i = 0; i < 3; i++) c[i] = base[i] * k;
    }
    for (int i = 0; i < 3; i++) rgb[i] = to_u8(c[i]);
    if (depth) *depth = t;
    if (label) *label = (unsigned char)lab;
}

}  // namespace render
}  // namespace uhc
