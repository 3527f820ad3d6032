// render_mesh_core.h -- the mesh renderer's per-frame refit and per-pixel cast (include/uhc_render.h uhc_render_mesh), for the device
// (render_mesh.cu) and, with -DUHC_EMU, for the host emulation the CPU tests run (tests/emu/render_mesh_emu.cpp).
//
// The scene is the skinned SMPL mesh of one or two humanoids under a fixed two-level hierarchy: body -> leaves of <= MESH_LEAF faces ->
// triangles.  The topology (the faces permuted so that every leaf is a contiguous run, body-major) is built once per model on the host
// (uhc_b200/render_mesh.py); per frame only the boxes are refitted.  The pixel path is render_core.h's shade_pixel with the overloads of
// cast and focus_xy below, under render_core.h's rule: fp32 + - * /, sqrt and floorf (and the exact min / max of the boxes) only, so a
// device build with -fmad=false and a host build with -ffp-contract=off give the same bits.
#pragma once
#include "render_core.h"

namespace uhc {
namespace render {

constexpr int MESH_LEAF = 32;                 // faces of a leaf, at most
constexpr float SLAB_PAD = 1.0000004f;        // a slab's far distance is widened by ~3.5 ulp: a box never loses a ray its faces would take

// the scene of one frame.  Boxes are [lo x y z, hi x y z]: body box of slot j = 24 h + b at body_box + 6 j, leaf box l of humanoid h at
// leaf_box + 6 (h nleaf + l).  verts[h] = the frame's [V][3] vertices of humanoid h, unshifted (the ghost is shifted by `shift` in x as it
// is read, with the same fp32 addition the refit uses).
struct MeshScene {
    const float *verts[2];
    const int *face;              // [F][3], permuted
    const int *leaf_first;        // [nleaf + 1]
    const int *body_leaf;         // [25]
    const float *body_box, *leaf_box;
    int nleaf, visible;
    float shift;
    const float *root;            // the first humanoid's root (x, y, z), where a focused camera looks
};

UHC_RDEV void focus_xy(const MeshScene &s, float *look) { look[0] = s.root[0]; look[1] = s.root[1]; }

UHC_RDEV float fmin_(float a, float b) { return b < a ? b : a; }
UHC_RDEV float fmax_(float a, float b) { return b > a ? b : a; }

// vertex k of humanoid h, the ghost shifted in x
UHC_RDEV void mesh_vertex(const MeshScene &s, int h, int k, float *v) {
    const float *p = (h ? s.verts[1] : s.verts[0]) + 3 * (size_t)k;
    v[0] = h ? p[0] + s.shift : p[0]; v[1] = p[1]; v[2] = p[2];
}

// ---- the refit: the box of leaf l's vertices (faces leaf_first[l] .. leaf_first[l + 1] - 1)
UHC_RDEV void refit_leaf(const float *verts, const int *face, int f0, int f1, int ghost, float shift, float *box) {
    float lo[3] = {INF, INF, INF}, hi[3] = {-INF, -INF, -INF};
    for (int f = f0; f < f1; f++)
        for (int c = 0; c < 3; c++) {
            const float *p = verts + 3 * (size_t)face[3 * f + c];
            const float v[3] = {ghost ? p[0] + shift : p[0], p[1], p[2]};
            for (int k = 0; k < 3; k++) { lo[k] = fmin_(lo[k], v[k]); hi[k] = fmax_(hi[k], v[k]); }
        }
    for (int k = 0; k < 3; k++) { box[k] = lo[k]; box[3 + k] = hi[k]; }
}
// the union of leaf boxes l0 .. l1 - 1.  A body without leaves gets the box at +inf on every bound, which slab never enters (every axis gives
// +inf or -inf at both ends, never NaN); an inverted box (+inf, -inf) would be entered by every ray, since slab orders each axis' ends.
UHC_RDEV void union_boxes(const float *leaf_box, int l0, int l1, float *box) {
    float b[6] = {INF, INF, INF, l0 < l1 ? -INF : INF, l0 < l1 ? -INF : INF, l0 < l1 ? -INF : INF};
    for (int l = l0; l < l1; l++)
        for (int k = 0; k < 3; k++) { b[k] = fmin_(b[k], leaf_box[6 * l + k]); b[3 + k] = fmax_(b[3 + k], leaf_box[6 * l + 3 + k]); }
    for (int k = 0; k < 6; k++) box[k] = b[k];
}

// ---- the pixel path
// slab test of the ray o + t d (inv = 1 / d per axis) against a box: does it meet the box for some t in [t_lo, t_hi)?
UHC_RDEV bool slab(const float *box, const float *o, const float *inv, float t_lo, float t_hi) {
    float t0 = t_lo, t1 = INF;
    for (int k = 0; k < 3; k++) {
        const float a = (box[k] - o[k]) * inv[k], b = (box[3 + k] - o[k]) * inv[k];
        if (a != a || b != b) continue;                         // 0 * inf: the ray runs in the plane of a face of the box
        t0 = fmax_(t0, fmin_(a, b)); t1 = fmin_(t1, fmax_(a, b));
    }
    return t0 <= t1 * SLAB_PAD && t0 < t_hi;
}

// watertight ray-triangle test (Woop, Benthin & Wald 2013, without the fp64 fall-back): the ray is sheared so that it runs along +z, and the
// edge functions U, V, W are computed from the sheared vertices alone, so two faces sharing an edge evaluate it to exactly opposite values
// and no ray passes between them.  kx, ky, kz and S come from the ray.  Returns t in (t_lo, t_hi), or -1 for a miss (a zero-area face:
// det = 0, never hit).
UHC_RDEV float pick(const float *v, int k) { return k == 0 ? v[0] : (k == 1 ? v[1] : v[2]); }   // v[k] without indexing by a variable
UHC_RDEV float tri_hit(const float *v0, const float *v1, const float *v2, const float *o, int kx, int ky, int kz, const float *S, float t_lo,
                       float t_hi) {
    const float A[3] = {v0[0] - o[0], v0[1] - o[1], v0[2] - o[2]};
    const float B[3] = {v1[0] - o[0], v1[1] - o[1], v1[2] - o[2]};
    const float C[3] = {v2[0] - o[0], v2[1] - o[1], v2[2] - o[2]};
    const float Az = pick(A, kz), Bz = pick(B, kz), Cz = pick(C, kz);
    const float Ax = pick(A, kx) - S[0] * Az, Ay = pick(A, ky) - S[1] * Az;
    const float Bx = pick(B, kx) - S[0] * Bz, By = pick(B, ky) - S[1] * Bz;
    const float Cx = pick(C, kx) - S[0] * Cz, Cy = pick(C, ky) - S[1] * Cz;
    const float U = Cx * By - Cy * Bx, V = Ax * Cy - Ay * Cx, W = Bx * Ay - By * Ax;
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return -1.0f;
    const float det = (U + V) + W;
    if (det == 0.0f) return -1.0f;
    const float T = (U * (S[2] * Az) + V * (S[2] * Bz)) + W * (S[2] * Cz);
    const float t = T / det;
    return (t > t_lo && t < t_hi) ? t : -1.0f;
}

// the ray o + t d (world, |d| = 1) against every visible humanoid's mesh, t in (t_lo, *t_best): the nearest hit's slot (-1: none), *t_best
// and the hit face's normal nw (unit, turned towards the ray's origin) updated.  any: stop at the first hit (shadow rays).
UHC_RDEV int cast(const MeshScene &s, const float *o, const float *d, float t_lo, float *t_best, float *nw, bool any) {
    const float inv[3] = {1.0f / d[0], 1.0f / d[1], 1.0f / d[2]};
    const float ax = d[0] < 0.0f ? -d[0] : d[0], ay = d[1] < 0.0f ? -d[1] : d[1], az = d[2] < 0.0f ? -d[2] : d[2];
    const int kz = (ax >= ay && ax >= az) ? 0 : (ay >= az ? 1 : 2);
    int kx = kz == 2 ? 0 : kz + 1, ky = kx == 2 ? 0 : kx + 1;
    if (pick(d, kz) < 0.0f) { const int k = kx; kx = ky; ky = k; }   // keeps the winding
    const float dz = pick(d, kz), S[3] = {pick(d, kx) / dz, pick(d, ky) / dz, 1.0f / dz};
    int hit = -1, hf = -1;
    for (int h = 0; h < 2; h++) {
        if (!((s.visible >> h) & 1)) continue;
        for (int b = 0; b < NB; b++) {
            const int j = h * NB + b;
            if (!slab(s.body_box + 6 * j, o, inv, t_lo, *t_best)) continue;
            for (int l = s.body_leaf[b]; l < s.body_leaf[b + 1]; l++) {
                if (!slab(s.leaf_box + 6 * ((size_t)h * s.nleaf + l), o, inv, t_lo, *t_best)) continue;
                for (int f = s.leaf_first[l]; f < s.leaf_first[l + 1]; f++) {
                    float v0[3], v1[3], v2[3];
                    mesh_vertex(s, h, s.face[3 * f], v0); mesh_vertex(s, h, s.face[3 * f + 1], v1); mesh_vertex(s, h, s.face[3 * f + 2], v2);
                    const float t = tri_hit(v0, v1, v2, o, kx, ky, kz, S, t_lo, *t_best);
                    if (t < 0.0f) continue;
                    *t_best = t; hit = j; hf = f;
                    if (any) return hit;
                }
            }
        }
    }
    if (hit >= 0) {
        const int h = hit / NB;
        float v0[3], v1[3], v2[3];
        mesh_vertex(s, h, s.face[3 * hf], v0); mesh_vertex(s, h, s.face[3 * hf + 1], v1); mesh_vertex(s, h, s.face[3 * hf + 2], v2);
        const float e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]}, e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
        float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
        const float nn = dot3(n, n);
        if (nn > 0.0f) {
            const float sg = dot3(n, d) > 0.0f ? -1.0f : 1.0f, k = sg / sqrtf(nn);
            for (int i = 0; i < 3; i++) nw[i] = n[i] * k;
        } else { nw[0] = -d[0]; nw[1] = -d[1]; nw[2] = -d[2]; }   // a face too thin for fp32's cross product: lit as if seen head-on
    }
    return hit;
}

#ifdef UHC_RENDER_HOST
// host only: the checks of uhc_render_mesh_init (0, or -2 with *why set)
inline int mesh_tables_check(const UhcRenderMesh &m, const char **why) {
    if (!m.face || !m.face_body || !m.leaf_first || !m.body_leaf) { *why = "null table"; return -2; }
    if (m.nvert < 3 || m.nface < 1 || m.nleaf < 1) { *why = "nvert >= 3, nface >= 1 and nleaf >= 1 are required"; return -2; }
    for (long i = 0; i < 3L * m.nface; i++)
        if (m.face[i] < 0 || m.face[i] >= m.nvert) { *why = "a face index is outside 0 .. nvert - 1"; return -2; }
    if (m.leaf_first[0] != 0 || m.leaf_first[m.nleaf] != m.nface) { *why = "the leaves do not cover the faces exactly once"; return -2; }
    for (int l = 0; l < m.nleaf; l++) {
        const int c = m.leaf_first[l + 1] - m.leaf_first[l];
        if (c < 1 || c > MESH_LEAF) { *why = "a leaf is empty or holds more than 32 faces"; return -2; }
    }
    if (m.body_leaf[0] != 0 || m.body_leaf[NB] != m.nleaf) { *why = "the bodies' leaf ranges do not cover the leaves"; return -2; }
    for (int b = 0; b < NB; b++)
        if (m.body_leaf[b + 1] < m.body_leaf[b]) { *why = "a body's leaves are not contiguous"; return -2; }
    for (int b = 0; b < NB; b++) {
        for (int f = m.leaf_first[m.body_leaf[b]]; f < m.leaf_first[m.body_leaf[b + 1]]; f++)
            if (m.face_body[f] != b) { *why = "a face lies in a leaf of another body"; return -2; }
    }
    return 0;
}
#endif

}  // namespace render
}  // namespace uhc
