// motion_core.h -- expert-table records built from raw motion, one frame per thread, in fp64.
//
// Restates uhc_b200/motion_lib.py (smpl_to_qpos + qpos_fk, which tests/test_motion_lib.py pins to the reference's
// smpl_to_qpose + Humanoid.qpos_fk) operation for operation, in the same evaluation order, so that a build without
// contracted multiply-adds (motion_lib.cu: -fmad=false; the host emulation: -ffp-contract=off) reproduces the numpy table
// to rounding of the math library.  Written like sim_core.h: the same source compiles as CUDA device code and, with
// -DUHC_EMU, as host code for the CPU tests (tests/emu).
//
// Record layout (include/uhc_b200.h UHC_EX_SIZE = 576):
//   qpos76 qvel75 wbpos72 wbquat96 bquat96 bangvel72 ee_wpos15 body_com72 (com = its first 3) pad2
// Finite differences (get_qvel_fd_batch, torch_utils.py:368-386) at dt = 1/30: the difference of frames t and t + 1 is stored
// at row t + 1 and row 0 repeats row 1.  The thread of row r recomputes the qpos of both frames of its difference from the
// raw input, so no difference is ever taken from a table that was rounded to the engine's precision.
#pragma once
#include <math.h>

#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_MDEV __device__ __forceinline__
#else
#define UHC_MDEV static inline
#endif

namespace uhc {
namespace motion {

constexpr int MB = 24, MQ = 76, MV = 75, REC = 576;
constexpr int KIND_SMPL = 0, KIND_QPOS = 1;   // include/uhc_b200.h UHC_MOTION_SMPL / UHC_MOTION_QPOS
constexpr int BODY6 = 6;                      // per body and shape variant: offset3 ipos3 (body_f columns 0:6, fp64)
constexpr int R_QPOS = 0, R_QVEL = 76, R_WBPOS = 151, R_WBQUAT = 223, R_BQUAT = 319, R_BANGVEL = 415, R_EE = 487, R_BCOM = 502, R_PAD = 574;

// the kinematic tables of the FK, passed by value
struct MotionModel {
    int parent[MB];       // bodies numbered depth-first: parent[b] < b
    int ee[5];            // end-effector bodies (ee_wpos)
    int smpl_joint[MB];   // SMPL joint (SMPL_BONE_ORDER_NAMES) of every model body
    const double *body;   // [nshape][MB][BODY6]; the root offset is body 0's offset (model.root_offset)
};

// SMPL_BONE_ORDER_NAMES.index(name) for name in model.body_names (uhc_b200/motion_lib.py smpl_to_qpos)
inline void motion_model_init(MotionModel &m, const int *parent, const int *ee, const double *body) {
    static const int order[MB] = {0, 1, 4, 7, 10, 2, 5, 8, 11, 3, 6, 9, 12, 15, 13, 16, 18, 20, 22, 14, 17, 19, 21, 23};
    for (int b = 0; b < MB; b++) { m.parent[b] = parent[b]; m.smpl_joint[b] = order[b]; }
    for (int i = 0; i < 5; i++) m.ee[i] = ee[i];
    m.body = body;
}
// fp64 columns 0:6 of the model's body_f ([nshape][24][UHC_BODYF]) -> [nshape][24][BODY6]
inline void motion_body_table(const double *body_f, int bodyf, int nshape, double *out) {
    for (int s = 0; s < nshape * MB; s++)
        for (int k = 0; k < BODY6; k++) out[(size_t)s * BODY6 + k] = body_f[(size_t)s * bodyf + k];
}

// ---- quaternion helpers, wxyz, in the evaluation order of motion_lib.py
UHC_MDEV void m_qmul(const double *a, const double *b, double *o) {
    const double w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
    const double x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
    const double y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
    const double z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
    o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}
UHC_MDEV void m_qinv(const double *q, double *o) {
    const double n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    o[0] = q[0] / n; o[1] = -q[1] / n; o[2] = -q[2] / n; o[3] = -q[3] / n;
}
UHC_MDEV void m_cross(const double *a, const double *b, double *o) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
// qrot(q, v) + p: v + 2 (w uv + uuv) + p
UHC_MDEV void m_qrot_add(const double *q, const double *v, const double *p, double *o) {
    double uv[3], uuv[3];
    m_cross(q + 1, v, uv); m_cross(q + 1, uv, uuv);
    for (int i = 0; i < 3; i++) o[i] = (v[i] + 2 * (q[0] * uv[i] + uuv[i])) + p[i];
}
// quaternion_from_euler(e0, e1, e2, 'rzyx') = Rz(e0) Ry(e1) Rx(e2) (euler_zyx_quat)
UHC_MDEV void m_euler_zyx_quat(const double *e, double *o) {
    double c[3], s[3];
    for (int i = 0; i < 3; i++) { const double h = 0.5 * e[i]; c[i] = cos(h); s[i] = sin(h); }
    const double qz[4] = {c[0], 0.0, 0.0, s[0]}, qy[4] = {c[1], 0.0, s[1], 0.0}, qx[4] = {c[2], s[2], 0.0, 0.0};
    double t[4];
    m_qmul(qz, qy, t); m_qmul(t, qx, o);
}
// rotation_from_quaternion_batch (torch_utils.py:142-167): axis and angle, with the arccos clamp and the |sin| < 1e-5 branch
UHC_MDEV void m_rot_from_quat(const double *q, double *axis, double *angle) {
    const double w = q[0] < -1.0 + 1e-7 ? -1.0 + 1e-7 : (q[0] > 1.0 - 1e-7 ? 1.0 - 1e-7 : q[0]);
    const double ac = acos(w), sn = sin(ac);
    if (fabs(sn) < 1e-5) { axis[0] = 1.0; axis[1] = 0.0; axis[2] = 0.0; *angle = 0.0; return; }
    for (int i = 0; i < 3; i++) axis[i] = q[1 + i] / sn;
    *angle = 2 * ac;
}

// ---- scipy.spatial.transform.Rotation, the steps smpl_to_qpos uses (quaternions xyzw here, as scipy stores them)
// from_rotvec, including the series below an angle of 1e-3
UHC_MDEV void m_rotvec_quat(const double *rv, double *q) {
    const double angle = sqrt(rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2]);
    double scale;
    if (angle <= 1e-3) { const double a2 = angle * angle; scale = 0.5 - a2 / 48 + a2 * a2 / 3840; }
    else scale = sin(angle / 2) / angle;
    q[0] = scale * rv[0]; q[1] = scale * rv[1]; q[2] = scale * rv[2]; q[3] = cos(angle / 2);
}
// as_euler("ZYX"): the quaternion algorithm of Bernardes & Viollet (2022) for the intrinsic sequence ZYX, i.e. the extrinsic axes
// i, j, k = x, y, z read backwards (even permutation, sign +1, lambda = pi / 2).  Second angle within 1e-7 of 0 or pi (gimbal lock):
// the third angle is set to 0 and the first takes the whole rotation about the remaining axis.  Output: angles about Z, Y, X.
UHC_MDEV void m_quat_euler_zyx(const double *q, double *ang) {
    const double pi = M_PI;
    const double a = q[3] - q[1], b = q[0] + q[2], c = q[1] + q[3], d = q[2] - q[0];
    double e[3];
    e[1] = 2 * atan2(hypot(c, d), hypot(a, b));
    const int cs = fabs(e[1]) <= 1e-7 ? 1 : (fabs(e[1] - pi) <= 1e-7 ? 2 : 0);
    const double half_sum = atan2(b, a), half_diff = atan2(d, c);
    if (cs == 0) { e[2] = half_sum - half_diff; e[0] = half_sum + half_diff; }
    else { e[2] = 0.0; e[0] = cs == 1 ? 2 * half_sum : 2 * half_diff; }
    e[1] -= pi / 2;
    for (int i = 0; i < 3; i++) {
        if (e[i] < -pi) e[i] += 2 * pi;
        else if (e[i] > pi) e[i] -= 2 * pi;
        ang[i] = e[i];
    }
}

// smpl_to_qpos of one frame.  row = pose_aa (72 | 156: columns 66:72 read as zero, smplh_to_smpl) then trans (3)
UHC_MDEV void m_smpl_qpos(const MotionModel &m, const double *row, int pose_dim, const double *root_off, double *qpos) {
    for (int b = 0; b < MB; b++) {
        const int j = m.smpl_joint[b];
        double rv[3], q[4];
        for (int k = 0; k < 3; k++) rv[k] = (pose_dim == 156 && j >= 22) ? 0.0 : row[3 * j + k];
        m_rotvec_quat(rv, q);
        if (b == 0) {   // root: the quaternion itself (wxyz, w >= 0)
            const double s = q[3] < 0 ? -1.0 : 1.0;
            qpos[3] = s * q[3]; qpos[4] = s * q[0]; qpos[5] = s * q[1]; qpos[6] = s * q[2];
        } else m_quat_euler_zyx(q, qpos + 7 + 3 * (b - 1));
    }
    for (int k = 0; k < 3; k++) qpos[k] = row[pose_dim + k] + root_off[k];
}
UHC_MDEV void m_load_qpos(const MotionModel &m, int kind, int pose_dim, const double *row, const double *root_off, double *qpos) {
    if (kind == KIND_QPOS) { for (int i = 0; i < MQ; i++) qpos[i] = row[i]; }
    else m_smpl_qpos(m, row, pose_dim, root_off, qpos);
}
// body-local quaternions (bquat): the root quaternion, then euler_zyx_quat of every hinge triple
UHC_MDEV void m_local_quats(const double *qpos, double *bq) {
    for (int k = 0; k < 4; k++) bq[k] = qpos[3 + k];
    for (int b = 1; b < MB; b++) m_euler_zyx_quat(qpos + 7 + 3 * (b - 1), bq + 4 * b);
}
// one step of the FK down the tree: body b's world position / quaternion from its parent's (the root's from qpos); body = the variant's
// [MB][BODY6] table, bq = m_local_quats of q.  Called for b = 0, 1, .. in order (motion_frame, and the renderer's pose pass).
UHC_MDEV void m_fk_body(const MotionModel &m, int b, const double *q, const double *bq, const double *body, double *wpos, double *wq) {
    if (b == 0) { for (int k = 0; k < 3; k++) wpos[k] = q[k]; for (int k = 0; k < 4; k++) wq[k] = q[3 + k]; }
    else {
        const int p = m.parent[b];
        m_qrot_add(wq + 4 * p, body + b * BODY6, wpos + 3 * p, wpos + 3 * b);
        m_qmul(wq + 4 * p, bq + 4 * b, wq + 4 * b);
    }
}

// The record of frame t of a clip whose rows start at `rows` (row width row_w); variant = the clip's body-shape variant.
template <class Out>
UHC_MDEV void motion_frame(const MotionModel &m, int kind, int pose_dim, const double *rows, int row_w, int t, int variant, Out *rec) {
    const double dt = 1.0 / 30;
    const double *body = m.body + (size_t)variant * MB * BODY6;
    // frames of the difference stored at row t: (t - 1, t), and (0, 1) for row 0
    const int fa = t > 0 ? t - 1 : 0, fb = t > 0 ? t : 1;
    double qa[MQ], qb[MQ], bqa[4 * MB], bqb[4 * MB];
    m_load_qpos(m, kind, pose_dim, rows + (size_t)fa * row_w, body, qa);
    m_load_qpos(m, kind, pose_dim, rows + (size_t)fb * row_w, body, qb);
    m_local_quats(qa, bqa); m_local_quats(qb, bqb);
    const double *q = t > 0 ? qb : qa, *bq = t > 0 ? bqb : bqa;
    for (int i = 0; i < MQ; i++) rec[R_QPOS + i] = (Out)q[i];
    {   // qvel: root linear velocity, root angular velocity in the root frame, hinge differences (not wrapped); clipped to +-10
        double v[MV];
        for (int i = 0; i < 3; i++) v[i] = (qb[i] - qa[i]) / dt;
        double inv[4], rel[4], axis[3], angle;
        m_qinv(qa + 3, inv); m_qmul(qb + 3, inv, rel);
        m_rot_from_quat(rel, axis, &angle);
        if (angle > M_PI) angle = angle - 2 * M_PI;
        if (angle < -M_PI) angle = angle + 2 * M_PI;
        double rv[3];
        for (int i = 0; i < 3; i++) rv[i] = axis[i] * angle / dt;
        // qmat(cur)^T rv, qmat normalising the quaternion first
        const double *c = qa + 3;
        const double nrm = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2] + c[3] * c[3]);
        const double w = c[0] / nrm, x = c[1] / nrm, y = c[2] / nrm, z = c[3] / nrm;
        const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                             2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                             2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
        for (int i = 0; i < 3; i++) v[3 + i] = R[i] * rv[0] + R[3 + i] * rv[1] + R[6 + i] * rv[2];
        for (int i = 6; i < MV; i++) v[i] = (qb[i + 1] - qa[i + 1]) / dt;
        for (int i = 0; i < MV; i++) {
            const double x_ = v[i] < -10.0 ? -10.0 : (v[i] > 10.0 ? 10.0 : v[i]);
            rec[R_QVEL + i] = (Out)x_;
        }
    }
    for (int b = 0; b < MB; b++) {   // bangvel: rotation vector of bquat[t+1] bquat[t]^-1 over dt, not clipped
        double inv[4], rel[4], axis[3], angle;
        m_qinv(bqa + 4 * b, inv); m_qmul(bqb + 4 * b, inv, rel);
        m_rot_from_quat(rel, axis, &angle);
        for (int i = 0; i < 3; i++) rec[R_BANGVEL + 3 * b + i] = (Out)(axis[i] * angle / dt);
    }
    // FK down the tree: world positions / quaternions, body centres of mass
    double wpos[3 * MB], wq[4 * MB];
    for (int b = 0; b < MB; b++) {
        m_fk_body(m, b, q, bq, body, wpos, wq);
        double com[3];
        m_qrot_add(wq + 4 * b, body + b * BODY6 + 3, wpos + 3 * b, com);
        for (int k = 0; k < 3; k++) { rec[R_WBPOS + 3 * b + k] = (Out)wpos[3 * b + k]; rec[R_BCOM + 3 * b + k] = (Out)com[k]; }
        for (int k = 0; k < 4; k++) { rec[R_WBQUAT + 4 * b + k] = (Out)wq[4 * b + k]; rec[R_BQUAT + 4 * b + k] = (Out)bq[4 * b + k]; }
    }
    for (int i = 0; i < 5; i++)
        for (int k = 0; k < 3; k++) rec[R_EE + 3 * i + k] = (Out)wpos[3 * m.ee[i] + k];
    rec[R_PAD] = (Out)0; rec[R_PAD + 1] = (Out)0;
}

#ifndef UHC_EMU
// motion_lib.cu: one thread per frame writes the records of the clips [c0, c1) (frames clip_adr[c0] .. clip_adr[c1] - 1 of the table,
// nf of them); rows = the raw rows of those clips only, fk_model = shape variant per clip (NULL: variant 0)
template <class Out>
cudaError_t launch_motion_frames(const MotionModel &m, int kind, int pose_dim, const double *rows, const int *clip_adr, const int *fk_model,
                                 int c0, int c1, int nf, Out *table, cudaStream_t st);
#endif

}  // namespace motion
}  // namespace uhc
