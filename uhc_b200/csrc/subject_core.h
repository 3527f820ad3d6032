// subject_core.h -- one subject's body from the shipped humanoid, in fp64 (include/uhc_subject.h uhc_subject_bodies).
//
// Per model body b the subject's body is the image of the shipped one under an affine map x -> A x + t of the body frame, evaluated from a
// basis that is affine in the shape vector beta: (A | t) = C_0 + sum_l beta_l C_{l+1}, and the body offset moves by D_0 + sum_l beta_l D_{l+1}
// (uhc_b200/subject_body.py fits both bases once per gender).  What follows from the map is closed-form:
//   hull vertices   h' = A h + t (a convex polytope stays convex, with the same hull graph)
//   mass            m' = m |det A|                           (density unchanged)
//   centre of mass  c' = A c + t
//   inertia         S = tr(I)/2 1 - I (second moments about the COM), S' = |det A| A S A^T, I' = tr(S') 1 - S'
// A body whose map is exactly (1 | 0) keeps its shipped mass properties bit for bit.  The derived columns follow uhc_b200/model.py: the
// bounding sphere of _pack (vertex centroid, largest distance * 1.0001 + 1e-6) and _invweight0's translational invweight trace(Jv M^-1 Jv^T)/3
// at qpos0, with M the 75 x 75 joint-space inertia (armature on the diagonal), through its Cholesky factor: trace(Jv M^-1 Jv^T) = |L^-1 Jv^T|^2.
//
// Every function computes one item (a body, a vertex, a matrix entry) from its inputs alone, so the result has the same bits whichever thread
// computes it.  Written like motion_core.h: CUDA device code, or host code under -DUHC_EMU for the CPU tests (tests/emu).  Compiled without
// contracted multiply-adds (subject.cu is in build.py's NO_FMA_SRCS; the emulation uses -ffp-contract=off).
#pragma once
#include <math.h>

#ifndef UHC_MDEV
#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_MDEV __device__ __forceinline__
#else
#define UHC_MDEV static inline
#endif
#endif

namespace uhc {
namespace subj {

constexpr int NB = 24, NV = 75, NBETA = 10, NTERM = NBETA + 1, MAPW = 12, BODYF = 20;
constexpr int NTRI = NV * (NV + 1) / 2;       // packed lower triangle of M / L: entry (i, j), j <= i, at i (i + 1) / 2 + j

UHC_MDEV int tri(int i, int j) { return i * (i + 1) / 2 + j; }

// (A | t) of one body: basis [11][12] (3 rows of A_i0 A_i1 A_i2 t_i), beta [10]
UHC_MDEV void eval_map(const double *basis, const double *beta, double *map) {
    for (int k = 0; k < MAPW; k++) {
        double x = basis[k];
        for (int l = 0; l < NBETA; l++) x = x + beta[l] * basis[(l + 1) * MAPW + k];
        map[k] = x;
    }
}

// the change of one body offset: basis [11][3]
UHC_MDEV void eval_offset(const double *basis, const double *beta, const double *shipped, double *off) {
    for (int c = 0; c < 3; c++) {
        double x = basis[c];
        for (int l = 0; l < NBETA; l++) x = x + beta[l] * basis[(l + 1) * 3 + c];
        off[c] = shipped[c] + x;
    }
}

UHC_MDEV void apply(const double *map, const double *x, double *y) {
    for (int i = 0; i < 3; i++) y[i] = map[4 * i] * x[0] + map[4 * i + 1] * x[1] + map[4 * i + 2] * x[2] + map[4 * i + 3];
}

UHC_MDEV double det3(const double *m) {
    return m[0] * (m[5] * m[10] - m[6] * m[9]) - m[1] * (m[4] * m[10] - m[6] * m[8]) + m[2] * (m[4] * m[9] - m[5] * m[8]);
}

UHC_MDEV bool is_identity(const double *m) {
    for (int i = 0; i < 3; i++)
        for (int k = 0; k < 4; k++)
            if (m[4 * i + k] != (k == i ? 1.0 : 0.0)) return false;
    return true;
}

// mass properties of one body: shipped row bf [20] (ipos 3:6, mass 6, inertia xx yy zz xy xz yz 7:13) -> out [20] columns 3:13
UHC_MDEV void mass_props(const double *map, const double *bf, double *out) {
    if (is_identity(map)) {
        for (int k = 3; k < 13; k++) out[k] = bf[k];
        return;
    }
    const double ad = fabs(det3(map));
    apply(map, bf + 3, out + 3);
    out[6] = bf[6] * ad;
    const double *q = bf + 7;
    const double I[9] = {q[0], q[3], q[4], q[3], q[1], q[5], q[4], q[5], q[2]};
    const double h = 0.5 * (I[0] + I[4] + I[8]);
    double S[9];
    for (int k = 0; k < 9; k++) S[k] = (k % 4 == 0 ? h : 0.0) - I[k];
    double AS[9], Sp[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) AS[3 * i + j] = map[4 * i] * S[j] + map[4 * i + 1] * S[3 + j] + map[4 * i + 2] * S[6 + j];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) Sp[3 * i + j] = ad * (AS[3 * i] * map[4 * j] + AS[3 * i + 1] * map[4 * j + 1] + AS[3 * i + 2] * map[4 * j + 2]);
    const double tr = Sp[0] + Sp[4] + Sp[8];
    out[7] = tr - Sp[0]; out[8] = tr - Sp[4]; out[9] = tr - Sp[8];
    out[10] = -Sp[1]; out[11] = -Sp[2]; out[12] = -Sp[5];
}

// bounding sphere of a body's mapped hull vertices v [k][3] as model.py _pack states it (numpy: mean over axis 0, norm over axis 1): out [4]
UHC_MDEV void sphere(const double *v, int k, double *out) {
    double c[3] = {0.0, 0.0, 0.0};
    for (int i = 0; i < k; i++)
        for (int d = 0; d < 3; d++) c[d] = c[d] + v[3 * i + d];
    for (int d = 0; d < 3; d++) c[d] = c[d] / (double)k;
    double r = 0.0;
    for (int i = 0; i < k; i++) {
        const double x = v[3 * i] - c[0], y = v[3 * i + 1] - c[1], z = v[3 * i + 2] - c[2];
        const double n = sqrt(x * x + y * y + z * z);
        r = n > r ? n : r;
    }
    for (int d = 0; d < 3; d++) out[d] = c[d];
    out[3] = r * 1.0001 + 1e-6;
}

// --- the joint-space inertia at qpos0 (every rotation the identity): body frames are world-aligned, dofs 0..2 root translation, 3..5 root
// rotation about x, y, z, then 3 hinges per body about z, y, x (dof 6 + 3 (b - 1) + k)
struct Rest {
    double gpos[NB][3], xipos[NB][3], mass[NB], inertia[NB][6];
    int parent[NB], sub_end[NB];
};

UHC_MDEV void axis_of(int d, double *a) {     // dof d >= 3: its rotation axis
    a[0] = a[1] = a[2] = 0.0;
    if (d < 6) a[d - 3] = 1.0;
    else a[2 - (d - 6) % 3] = 1.0;
}

UHC_MDEV int body_of(int d) { return d < 6 ? 0 : 1 + (d - 6) / 3; }

// column d of body b's translational / rotational Jacobian at its COM; false when the dof does not move the body
UHC_MDEV bool jac(const Rest &R, int b, int d, double *jv, double *jw) {
    if (d < 3) {
        jv[0] = jv[1] = jv[2] = 0.0; jv[d] = 1.0;
        jw[0] = jw[1] = jw[2] = 0.0;
        return true;
    }
    const int a = body_of(d);
    if (d >= 6 && !(a <= b && b <= R.sub_end[a])) return false;
    double ax[3];
    axis_of(d, ax);
    const double r[3] = {R.xipos[b][0] - R.gpos[a][0], R.xipos[b][1] - R.gpos[a][1], R.xipos[b][2] - R.gpos[a][2]};
    jv[0] = ax[1] * r[2] - ax[2] * r[1]; jv[1] = ax[2] * r[0] - ax[0] * r[2]; jv[2] = ax[0] * r[1] - ax[1] * r[0];
    jw[0] = ax[0]; jw[1] = ax[1]; jw[2] = ax[2];
    return true;
}

// M[i][j], j <= i: armature on the diagonal + sum over bodies of m Jv_i . Jv_j + Jw_i . I Jw_j
UHC_MDEV double m_entry(const Rest &R, const double *armature, int i, int j) {
    double s = i == j ? armature[i] : 0.0;
    for (int b = 0; b < NB; b++) {
        double vi[3], wi[3], vj[3], wj[3];
        if (!jac(R, b, i, vi, wi) || !jac(R, b, j, vj, wj)) continue;
        const double *q = R.inertia[b];
        const double Iw[3] = {q[0] * wj[0] + q[3] * wj[1] + q[4] * wj[2], q[3] * wj[0] + q[1] * wj[1] + q[5] * wj[2],
                              q[4] * wj[0] + q[5] * wj[1] + q[2] * wj[2]};
        s = s + R.mass[b] * (vi[0] * vj[0] + vi[1] * vj[1] + vi[2] * vj[2]) + (wi[0] * Iw[0] + wi[1] * Iw[1] + wi[2] * Iw[2]);
    }
    return s;
}

// right-looking Cholesky of the packed M in place, column k: the pivot, then the column below it, then one entry (i, j), k < j <= i, of
// the trailing update.  Callers run the three steps in this order, every entry of a step before the next step.
UHC_MDEV void chol_pivot(double *L, int k) { L[tri(k, k)] = sqrt(L[tri(k, k)]); }
UHC_MDEV void chol_col(double *L, int k, int i) { L[tri(i, k)] = L[tri(i, k)] / L[tri(k, k)]; }
UHC_MDEV void chol_update(double *L, int k, int i, int j) { L[tri(i, j)] = L[tri(i, j)] - L[tri(i, k)] * L[tri(j, k)]; }

// |L^-1 Jv_b[c]^T|^2 for body b and translational component c; y [75] is scratch
UHC_MDEV double invw_part(const Rest &R, const double *L, int b, int c, double *y) {
    double s = 0.0;
    for (int i = 0; i < NV; i++) {
        double jv[3], jw[3];
        double x = jac(R, b, i, jv, jw) ? jv[c] : 0.0;
        for (int k = 0; k < i; k++) x = x - L[tri(i, k)] * y[k];
        y[i] = x / L[tri(i, i)];
        s = s + y[i] * y[i];
    }
    return s;
}

}  // namespace subj
}  // namespace uhc
