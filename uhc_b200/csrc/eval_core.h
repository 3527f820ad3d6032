// eval_core.h -- per-frame imitation metrics of one environment, in fp64.
//
// Restates uhc_b200/metrics.py (compute_metrics, procrustes_mpjpe, root_dist_mm; pinned to the reference's smpl_eval.compute_metrics
// by tests/test_metrics.py) for ONE recorded frame k of one episode, in the same evaluation order, so that a build without contracted
// multiply-adds (eval.cu: -fmad=false; the host emulation: -ffp-contract=off) agrees with numpy to the rounding of the SVD.
// Written like motion_core.h: the same source compiles as CUDA device code and, with -DUHC_EMU, as host code for the CPU tests.
//
// Inputs per frame: pred = the simulated qpos (root pos + quat: its first 7 values) and world joint positions xpos [24][3]; gt = the
// expert qpos / wbpos of the frame.  Output (EV_* columns), all per frame:
//   mpjpe_g   mean_j |pred_j - gt_j| * 1000                                   (mm)
//   mpjpe     the same after subtracting joint 0 (Pelvis) from each set        (mm)
//   pa_mpjpe  the same after the similarity (Procrustes) alignment of pred onto gt, root-relative sets   (mm)
//   vel       frame k >= 1: mean_j |(p_k - p_{k-1}) - (g_k - g_{k-1})| * 1000                            (mm)
//   accel     frame k >= 2: mean_j |(p_{k-2} - 2 p_{k-1} + p_k) - (g_{k-2} - 2 g_{k-1} + g_k)| * 1000    (mm)
//   root      |I - X_pred X_gt^-1|_F of the root transforms, BEFORE root_dist_mm's division by the number of frames and its * 1000
//             (the count is known only when the episode has ended; the caller applies  / T * 1000.0  in that order)
#pragma once
#include <math.h>

#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_EDEV __device__ __forceinline__
#else
#define UHC_EDEV static inline
#endif

namespace uhc {
namespace evalm {

constexpr int EJ = 24;                        // joints (SMPL bodies)
constexpr int EV_MPJPE_G = 0, EV_MPJPE = 1, EV_PA = 2, EV_VEL = 3, EV_ACCEL = 4, EV_ROOT = 5, EV_N = 6;

// numpy's pairwise sum of 24 contiguous values (.mean(-1) of a [T, 24] array): eight running sums, then ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7))
UHC_EDEV double sum24(const double *a) {
    double r[8];
    for (int i = 0; i < 8; i++) r[i] = a[i];
    for (int i = 8; i < EJ; i += 8)
        for (int j = 0; j < 8; j++) r[j] += a[i + j];
    return ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
}
UHC_EDEV double norm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }

// quat_to_mat4: rotation of (w, x, y, z) normalised by |q|^2 (identity when |q|^2 <= 4 eps)
UHC_EDEV void quat_mat3(const double *q, double M[3][3]) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double n = ((w * w + x * x) + y * y) + z * z;
    const double eps4 = 2.220446049250313e-16 * 4.0;
    if (!(n > eps4)) {
        for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) M[a][b] = a == b ? 1.0 : 0.0;
        return;
    }
    const double s = 2.0 / n;
    M[0][0] = 1 - s * (y * y + z * z); M[0][1] = s * (x * y - z * w); M[0][2] = s * (x * z + y * w);
    M[1][0] = s * (x * y + z * w); M[1][1] = 1 - s * (x * x + z * z); M[1][2] = s * (y * z - x * w);
    M[2][0] = s * (x * z - y * w); M[2][1] = s * (y * z + x * w); M[2][2] = 1 - s * (x * x + y * y);
}

// |I - X_p X_g^-1|_F with X = [R t; 0 1]: X_g^-1 = [R_g^T, -R_g^T t_g] (R_g is orthogonal by construction)
UHC_EDEV double root_fro(const double *qp, const double *qg) {
    double Rp[3][3], Rg[3][3];
    quat_mat3(qp + 3, Rp); quat_mat3(qg + 3, Rg);
    double acc = 0.0, RR[3][3];
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) {
            RR[a][b] = (Rp[a][0] * Rg[b][0] + Rp[a][1] * Rg[b][1]) + Rp[a][2] * Rg[b][2];
            const double e = (a == b ? 1.0 : 0.0) - RR[a][b];
            acc += e * e;
        }
    for (int a = 0; a < 3; a++) {      // translation column of X_p X_g^-1: t_p - R_p R_g^T t_g
        const double e = -(qp[a] - ((RR[a][0] * qg[0] + RR[a][1] * qg[1]) + RR[a][2] * qg[2]));
        acc += e * e;
    }
    return sqrt(acc);
}

// unit vector orthogonal to the unit vector u (cross product with the axis u is least aligned with)
UHC_EDEV void any_orthogonal(const double *u, double *o) {
    const double ax = fabs(u[0]), ay = fabs(u[1]), az = fabs(u[2]);
    double e[3] = {0.0, 0.0, 0.0};
    e[(ax <= ay && ax <= az) ? 0 : (ay <= az ? 1 : 2)] = 1.0;
    o[0] = u[1] * e[2] - u[2] * e[1]; o[1] = u[2] * e[0] - u[0] * e[2]; o[2] = u[0] * e[1] - u[1] * e[0];
    const double n = norm3(o[0], o[1], o[2]);
    for (int i = 0; i < 3; i++) o[i] /= n;
}

// procrustes_mpjpe of one frame: p, g = root-relative joint sets [24][3].  The SVD of H = G^T P is a one-sided Jacobi SVD
// (H V = U S, V a product of plane rotations), columns sorted by singular value.  numpy's reflection fix -- negate the last column of
// V and the last singular value when det(V U^T) < 0 -- is applied as R = V diag(1, 1, d) U^T, scale = (s1 + s2 + d s3) |G| / |P| with
// u3 = u1 x u2 and s3 = u3 . (H v3) signed: that product and that sum do not depend on the signs an SVD picks for its vectors.
// Rank-deficient H (every joint on one line, or a plane through the origin) leaves u2 / u3 free: u2 is then any unit vector
// orthogonal to u1, which changes nothing where P has no component along v2 / v3 (both sets on one line, or pred == gt).
UHC_EDEV double pa_mpjpe_frame(const double (*p)[3], const double (*g)[3]) {
    double mp[3] = {0.0, 0.0, 0.0}, mg[3] = {0.0, 0.0, 0.0};     // .mean(1) of [T, 24, 3]: a running sum over the joints
    for (int j = 0; j < EJ; j++)
        for (int c = 0; c < 3; c++) { mp[c] += p[j][c]; mg[c] += g[j][c]; }
    for (int c = 0; c < 3; c++) { mp[c] /= EJ; mg[c] /= EJ; }
    double sp = 0.0, sg = 0.0;
    for (int j = 0; j < EJ; j++)
        for (int c = 0; c < 3; c++) { const double a = p[j][c] - mp[c], b = g[j][c] - mg[c]; sp += a * a; sg += b * b; }
    const double np_ = sqrt(sp), ng = sqrt(sg);
    double W[3][3];                     // H = (G/|G|)^T (P/|P|), then rotated in place into U S
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) {
            double h = 0.0;
            for (int j = 0; j < EJ; j++) h += ((g[j][a] - mg[a]) / ng) * ((p[j][b] - mp[b]) / np_);
            W[a][b] = h;
        }
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 40; sweep++) {
        bool rotated = false;
        for (int pq = 0; pq < 3; pq++) {
            const int i = pq == 2 ? 1 : 0, k = pq == 0 ? 1 : 2;
            double al = 0.0, be = 0.0, ga = 0.0;
            for (int r = 0; r < 3; r++) { al += W[r][i] * W[r][i]; be += W[r][k] * W[r][k]; ga += W[r][i] * W[r][k]; }
            if (!(fabs(ga) > 1e-17 * sqrt(al * be)) || ga == 0.0) continue;
            rotated = true;
            const double zeta = (be - al) / (2.0 * ga);
            const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
            for (int r = 0; r < 3; r++) {
                const double wi = W[r][i], wk = W[r][k];
                W[r][i] = cs * wi - sn * wk; W[r][k] = sn * wi + cs * wk;
                const double vi = V[r][i], vk = V[r][k];
                V[r][i] = cs * vi - sn * vk; V[r][k] = sn * vi + cs * vk;
            }
        }
        if (!rotated) break;
    }
    double s[3];
    int ord[3] = {0, 1, 2};
    for (int c = 0; c < 3; c++) s[c] = norm3(W[0][c], W[1][c], W[2][c]);
    for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2 - a; b++)
            if (s[ord[b]] < s[ord[b + 1]]) { const int tmp = ord[b]; ord[b] = ord[b + 1]; ord[b + 1] = tmp; }
    double u[3][3], v[3][3], sv[3];      // u[i], v[i]: i-th singular vectors
    for (int i = 0; i < 3; i++) { sv[i] = s[ord[i]]; for (int r = 0; r < 3; r++) v[i][r] = V[r][ord[i]]; }
    for (int r = 0; r < 3; r++) u[0][r] = W[r][ord[0]] / sv[0];
    if (sv[1] > 1e-13 * sv[0]) for (int r = 0; r < 3; r++) u[1][r] = W[r][ord[1]] / sv[1];
    else {
        any_orthogonal(u[0], u[1]);
        sv[1] = (u[1][0] * W[0][ord[1]] + u[1][1] * W[1][ord[1]]) + u[1][2] * W[2][ord[1]];
    }
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1]; u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2]; u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    sv[2] = (u[2][0] * W[0][ord[2]] + u[2][1] * W[1][ord[2]]) + u[2][2] * W[2][ord[2]];
    // det(V U^T) = det(V) det(U), det(U) = +1 (u3 = u1 x u2)
    const double detv = v[0][0] * (v[1][1] * v[2][2] - v[1][2] * v[2][1]) - v[1][0] * (v[0][1] * v[2][2] - v[0][2] * v[2][1]) + v[2][0] * (v[0][1] * v[1][2] - v[0][2] * v[1][1]);
    const double d = detv > 0 ? 1.0 : (detv < 0 ? -1.0 : 0.0);
    double R[3][3];
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) R[a][b] = (v[0][a] * u[0][b] + v[1][a] * u[1][b]) + d * v[2][a] * u[2][b];
    const double scale = ((sv[0] + sv[1]) + d * sv[2]) * ng / np_;
    double mpR[3], err[EJ];
    for (int b = 0; b < 3; b++) mpR[b] = (mp[0] * R[0][b] + mp[1] * R[1][b]) + mp[2] * R[2][b];
    for (int j = 0; j < EJ; j++) {
        double e[3];
        for (int b = 0; b < 3; b++) {
            const double pr = (p[j][0] * R[0][b] + p[j][1] * R[1][b]) + p[j][2] * R[2][b];
            e[b] = (scale * pr + (mg[b] - scale * mpR[b])) - g[j][b];
        }
        err[j] = norm3(e[0], e[1], e[2]);
    }
    return sum24(err) / EJ;
}

// the six values of one frame.  pq / gq: qpos (the first 7 values are read), pj / gj: joint positions [72]; pj1, gj1 (pj2, gj2): the
// previous (second previous) recorded frame's joints, NULL where the episode has fewer frames (vel / accel are then 0)
UHC_EDEV void eval_frame(const double *pq, const double *gq, const double *pj, const double *gj, const double *pj1, const double *gj1,
                         const double *pj2, const double *gj2, double *out) {
    double d[EJ];
    for (int j = 0; j < EJ; j++) d[j] = norm3(pj[3 * j] - gj[3 * j], pj[3 * j + 1] - gj[3 * j + 1], pj[3 * j + 2] - gj[3 * j + 2]);
    out[EV_MPJPE_G] = sum24(d) / EJ * 1000.0;
    double pr[EJ][3], gr[EJ][3];
    for (int j = 0; j < EJ; j++)
        for (int c = 0; c < 3; c++) { pr[j][c] = pj[3 * j + c] - pj[c]; gr[j][c] = gj[3 * j + c] - gj[c]; }
    out[EV_PA] = pa_mpjpe_frame(pr, gr) * 1000.0;
    for (int j = 0; j < EJ; j++) d[j] = norm3(pr[j][0] - gr[j][0], pr[j][1] - gr[j][1], pr[j][2] - gr[j][2]);
    out[EV_MPJPE] = sum24(d) / EJ * 1000.0;
    out[EV_VEL] = 0.0;
    if (pj1) {
        for (int j = 0; j < EJ; j++) {
            double e[3];
            for (int c = 0; c < 3; c++) { const int i = 3 * j + c; e[c] = (pj[i] - pj1[i]) - (gj[i] - gj1[i]); }
            d[j] = norm3(e[0], e[1], e[2]);
        }
        out[EV_VEL] = sum24(d) / EJ * 1000.0;
    }
    out[EV_ACCEL] = 0.0;
    if (pj2) {
        for (int j = 0; j < EJ; j++) {
            double e[3];
            for (int c = 0; c < 3; c++) { const int i = 3 * j + c; e[c] = ((pj2[i] - 2 * pj1[i]) + pj[i]) - ((gj2[i] - 2 * gj1[i]) + gj[i]); }
            d[j] = norm3(e[0], e[1], e[2]);
        }
        out[EV_ACCEL] = sum24(d) / EJ * 1000.0;
    }
    out[EV_ROOT] = root_fro(pq, gq);
}

}  // namespace evalm
}  // namespace uhc
