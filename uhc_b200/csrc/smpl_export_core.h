// smpl_export_core.h -- qpos -> SMPL pose / translation, one frame per thread, in fp64: the inverse of motion_core.h's smpl_to_qpos.
//
// Restates the reference's qpos_to_smpl (uhc/smpllib/smpl_mujoco.py:738-752) exactly as it runs, through the scipy 1.18 calls it makes:
//   root:          Rotation.from_quat(q[[1, 2, 3, 0]]).as_rotvec()      (from_quat divides by the 4-norm; as_rotvec negates w < 0)
//   23 hinges:     Rotation.from_euler("ZYX", e).as_rotvec()            (elementary quaternions composed intrinsically)
//   trans:         qpos[0:3] - root offset                               (mj_model.body_pos[1]; here the frame's own shape variant)
// in the evaluation order of scipy's compiled (Cython) backend, which numpy arrays of this shape take, so a build without contracted
// multiply-adds (export.cu: -fmad=false; the host emulation: -ffp-contract=off) reproduces scipy to the rounding of the math library.
// Written like motion_core.h: the same source compiles as CUDA device code and, with -DUHC_EMU, as host code for the CPU tests.
//
// Output row (UHC_EVAL_SMPL = 75): pose 72 in SMPL_BONE_ORDER_NAMES order, then trans 3.
#pragma once
#include <math.h>
#include "motion_core.h"
#ifndef UHC_EMU
#include "../../include/uhc_eval.h"
#endif

namespace uhc {
namespace smplx {

constexpr int POSE = 72, ROW = 75;
using motion::MB;
using motion::BODY6;

// SMPL joint (SMPL_BONE_ORDER_NAMES index) of every model body: motion_core.h's order table, whose inverse the output order is
UHC_MDEV int smpl_joint_of(int b) {
    constexpr int order[MB] = {0, 1, 4, 7, 10, 2, 5, 8, 11, 3, 6, 9, 12, 15, 13, 16, 18, 20, 22, 14, 17, 19, 21, 23};
    return order[b];
}

// as_rotvec of one quaternion (xyzw): w < 0 -> -q, angle = 2 atan2(|v|, w), the series below an angle of 1e-3
UHC_MDEV void x_quat_rotvec(const double *q_in, double *rv) {
    double q[4];
    const double s = q_in[3] < 0 ? -1.0 : 1.0;
    for (int k = 0; k < 4; k++) q[k] = s < 0 ? -q_in[k] : q_in[k];
    const double angle = 2 * atan2(sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]), q[3]);
    double scale;
    if (angle <= 1e-3) { const double a2 = angle * angle; scale = 2 + a2 / 12 + 7 * a2 * a2 / 2880; }
    else scale = angle / sin(angle / 2);
    rv[0] = scale * q[0]; rv[1] = scale * q[1]; rv[2] = scale * q[2];
}
// scipy's compose_quat(p, q) (xyzw)
UHC_MDEV void x_compose(const double *p, const double *q, double *o) {
    const double c0 = p[1] * q[2] - p[2] * q[1], c1 = p[2] * q[0] - p[0] * q[2], c2 = p[0] * q[1] - p[1] * q[0];
    const double x = p[3] * q[0] + q[3] * p[0] + c0;
    const double y = p[3] * q[1] + q[3] * p[1] + c1;
    const double z = p[3] * q[2] + q[3] * p[2] + c2;
    const double w = p[3] * q[3] - p[0] * q[0] - p[1] * q[1] - p[2] * q[2];
    o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
// from_euler("ZYX", e): elementary quaternions about z, y, x (cos(a / 2) in w, sin(a / 2) on the axis), composed left to right
UHC_MDEV void x_euler_zyx(const double *e, double *q) {
    const int axis[3] = {2, 1, 0};
    double t[4];
    for (int i = 0; i < 3; i++) {
        double el[4] = {0.0, 0.0, 0.0, cos(e[i] / 2.0)};
        el[axis[i]] = sin(e[i] / 2.0);
        if (i == 0) for (int k = 0; k < 4; k++) q[k] = el[k];
        else { x_compose(q, el, t); for (int k = 0; k < 4; k++) q[k] = t[k]; }
    }
}

// One frame: qpos (76, any real type, read as double) -> out[0:72] pose, out[72:75] trans; root_off = the variant's root offset (3)
template <class Real>
UHC_MDEV void qpos_to_smpl(const Real *qpos, const double *root_off, double *out) {
    {   // root: from_quat of (x, y, z, w), divided by its 4-norm
        const double w = (double)qpos[3], x = (double)qpos[4], y = (double)qpos[5], z = (double)qpos[6];
        const double n = sqrt(x * x + y * y + z * z + w * w);
        const double q[4] = {x / n, y / n, z / n, w / n};
        x_quat_rotvec(q, out);
    }
    for (int b = 1; b < MB; b++) {
        double e[3], q[4];
        for (int k = 0; k < 3; k++) e[k] = (double)qpos[7 + 3 * (b - 1) + k];
        x_euler_zyx(e, q);
        x_quat_rotvec(q, out + 3 * smpl_joint_of(b));
    }
    for (int k = 0; k < 3; k++) out[POSE + k] = (double)qpos[k] - root_off[k];
}

#ifndef UHC_EMU
// export.cu: frames i < n, frame i's qpos at qpos + i * pitch (Real = float | double); variant[i] (NULL: 0) selects the root offset
// body[variant][0][0:3] of motion_core.h's body table; pose [n][72] and trans [n][3].  Arguments are the caller's to validate.
cudaError_t launch_qpos_to_smpl(const void *qpos, int precision, long n, long pitch, const int *variant, const double *body,
                                double *pose, double *trans, cudaStream_t st);
// export.cu, captured by eval.cu: k_eval_export over envs i < n (engine state / istate of that precision, clip_model per clip or NULL),
// window rows win_smpl[i][slot][ROW]; done = [n] frames already exported, zeroed at every reset.  Capturable.
cudaError_t launch_eval_export(int precision, const void *state, const int *istate, const int *clip_model, const double *body, const UhcEvalClip *clips,
                               int *done, int n, int window, int slot, double *win_smpl, cudaStream_t st);
#endif

}  // namespace smplx
}  // namespace uhc
