// floor_core.h -- the body hulls against the floor z = 0 (include/uhc_floor.h), per frame, in fp64: the lowest hull vertex, the mean depth of
// the vertices below the floor (compute_penetration, uhc/smpllib/smpl_eval.py:125-135, floor_z = 0), the mean horizontal travel of the
// vertices on the floor in two consecutive frames (compute_skate, :138-149) and the height of the lowest vertex above it.  The reference
// takes these from SMPL mesh vertices; here the surface is the convex hulls of the 24 collision bodies, the surface the simulator collides.
//
// The same source compiles as CUDA device code (floor.cu: -fmad=false) and, with -DUHC_EMU, as host code for the CPU tests
// (tests/emu/floor_emu.cpp: -ffp-contract=off).  A frame is one warp's work and its reduction order is fixed, so the host build gives the
// device's bits wherever the math library does (sin / cos of the pose pass):
//   1. place: qpos -> world rotation and position of every body, the renderer's pose pass (render_core.h pose_fk + pose_rows, which is
//      motion_core.h's FK); one lane per frame of the pair (t, t - 1)
//   2. lane_part: lane l takes vertices l, l + 32, .. in vertex order: world = R v + p, then its partial minimum, sums and counts
//   3. part_merge in a butterfly over lane distances 16, 8, 4, 2, 1; every merge is commutative, so all lanes end with lane 0's value
//   4. finish: the five columns
#pragma once
#include <math.h>
#include "render_core.h"

#ifndef UHC_EMU
#include "../../include/uhc_eval.h"
#define UHC_FDEV __device__ __forceinline__
#else
#define UHC_FDEV static inline
#endif

namespace uhc {
namespace floorm {

constexpr int NCOL = 5, LANES = 32, NFEET = 4;
constexpr int C_MINZ = 0, C_PEN = 1, C_SKATE = 2, C_FLOAT = 3, C_NBELOW = 4;   // include/uhc_floor.h UHC_FLOOR_NCOL
constexpr int POSE_ROW = render::NB * render::POSE;                            // one frame's body poses, doubles
constexpr double HUGE_Z = __builtin_huge_val();

// the hull vertices of one shape variant: vert = [nvert][3] in body frame, body[v] = the body vertex v belongs to
struct Hull { const double *vert; const unsigned char *body; int nvert; };

// a lane's share of a frame, and the merged value
struct Part { double min_z, below, skate; int n_below, n_skate; };

// L_Ankle, R_Ankle, L_Toe, R_Toe in the model's depth-first body order: the joints the reference's height rules read
// (uhc/data_process/process_amass_db.py:126-192)
UHC_FDEV int foot_body(int k) { return k == 0 ? 3 : (k == 1 ? 7 : (k == 2 ? 4 : 8)); }

// step 1: body poses [24][12] (R row-major, then the position) of one qpos with the variant's body table
UHC_FDEV void place(const motion::MotionModel &m, const double *q, const double *body, double *pose) {
    double wpos[3 * motion::MB], wq[4 * motion::MB];
    render::pose_fk(m, q, body, wpos, wq);
    render::pose_rows<double>(wpos, wq, pose);
}

UHC_FDEV void world_vertex(const double *P, const double *v, double *w) {
    for (int i = 0; i < 3; i++) w[i] = ((P[3 * i] * v[0] + P[3 * i + 1] * v[1]) + P[3 * i + 2] * v[2]) + P[9 + i];
}

// step 2; prev = the poses of the previous frame, or null
UHC_FDEV void lane_part(const Hull &h, const double *cur, const double *prev, int lane, Part *out) {
    Part p; p.min_z = HUGE_Z; p.below = 0.0; p.skate = 0.0; p.n_below = 0; p.n_skate = 0;
    for (int v = lane; v < h.nvert; v += LANES) {
        const int b = h.body[v];
        double w[3];
        world_vertex(cur + render::POSE * b, h.vert + 3 * v, w);
        if (w[2] < p.min_z) p.min_z = w[2];
        if (w[2] < 0.0) { p.below = p.below + w[2]; p.n_below++; }
        if (prev && w[2] <= 0.0) {
            double u[3];
            world_vertex(prev + render::POSE * b, h.vert + 3 * v, u);
            if (u[2] <= 0.0) {
                const double dx = w[0] - u[0], dy = w[1] - u[1];
                p.skate = p.skate + sqrt(dx * dx + dy * dy);
                p.n_skate++;
            }
        }
    }
    *out = p;
}

// step 3: a + b == b + a and the minimum of two numbers does not depend on their order
UHC_FDEV void part_merge(Part *a, const Part &b) {
    a->min_z = b.min_z < a->min_z ? b.min_z : a->min_z;
    a->below = a->below + b.below; a->skate = a->skate + b.skate;
    a->n_below += b.n_below; a->n_skate += b.n_skate;
}

// step 4: min_z (m), pen_mm, skate_mm (0 without a previous frame), float_mm, n_below
UHC_FDEV void finish(const Part &p, double *out) {
    out[C_MINZ] = p.min_z;
    out[C_PEN] = p.n_below ? -(p.below / (double)p.n_below) * 1000.0 : 0.0;
    out[C_SKATE] = p.n_skate ? (p.skate / (double)p.n_skate) * 1000.0 : 0.0;
    out[C_FLOAT] = (p.min_z > 0.0 ? p.min_z : 0.0) * 1000.0;
    out[C_NBELOW] = (double)p.n_below;
}

#ifdef UHC_EMU
// one frame as the warp computes it: q_prev = the previous frame's qpos, or null
static inline void frame_rows(const motion::MotionModel &m, const Hull &h, const double *body, const double *q, const double *q_prev, double *out,
                              double *feet) {
    double cur[POSE_ROW], prev[POSE_ROW];
    place(m, q, body, cur);
    if (q_prev) place(m, q_prev, body, prev);
    Part p[LANES], n[LANES];
    for (int l = 0; l < LANES; l++) lane_part(h, cur, q_prev ? prev : nullptr, l, &p[l]);
    for (int off = LANES / 2; off > 0; off >>= 1) {
        for (int l = 0; l < LANES; l++) { n[l] = p[l]; part_merge(&n[l], p[l ^ off]); }
        for (int l = 0; l < LANES; l++) p[l] = n[l];
    }
    finish(p[0], out);
    if (feet) for (int k = 0; k < NFEET; k++) feet[k] = cur[render::POSE * foot_body(k) + 11];
}
#endif

#ifndef UHC_EMU
// floor.cu, for the evaluation (eval.cu).  floor_gen: 0 before uhc_floor_init has run for this engine, else a number no other upload of
// hull vertices ever had: a graph that holds their device pointers carries it in its key.  launch_eval_floor, captured after
// k_eval_frame and before any fail_safe re-seat: one warp per env i < n that recorded a frame in this step (its clips[i].frames grew past
// done[i]) measures the state just recorded against prev[i] (the qpos of its previous recorded frame, [n][76] doubles, which it then
// replaces) into window row win_floor[i][slot][NCOL]; done / prev are zeroed / unspecified at every reset.  Capturable.
unsigned long long floor_gen(const UhcEngine *e);
cudaError_t launch_eval_floor(UhcEngine *e, int precision, const void *state, const int *istate, const int *clip_model, const UhcEvalClip *clips,
                              int *done, double *prev, int n, int window, int slot, double *win_floor, cudaStream_t st);
#endif

}  // namespace floorm
}  // namespace uhc
