// mesh_core.h -- the per-row half of the SMPL linear blend skinning (include/uhc_mesh.h), in fp64, as smplx's lbs states it:
//   rodrigues   batch_rodrigues: angle = |r + 1e-8|, axis = r / angle, R = I + sin K + (1 - cos) K^2
//   row_chain   the pose feature (R_k - I, k = 1 .. 23, row-major), batch_rigid_transform's chain G_k = G_parent [R_k | J_k - J_parent] and its
//               A_k = G_k - pad(G_k J_k), and the posed joints G_k.t + trans
// The per-vertex half (the pose blend and the skinning sum, in fp32) is in mesh.cu.  Device code; sm_90a.
#pragma once
#include <math.h>

namespace uhc {
namespace meshm {

constexpr int NJ = 24, NPF = 207, NBETA = 10;
constexpr int AROW = 12;               // A_k per joint: rows i = 0 .. 2 of [R | t] as (R_i0, R_i1, R_i2, t_i)

__device__ __forceinline__ void rodrigues(const double *r, double *R) {
    const double a0 = r[0] + 1e-8, a1 = r[1] + 1e-8, a2 = r[2] + 1e-8;
    const double ang = sqrt(a0 * a0 + a1 * a1 + a2 * a2);
    const double x = r[0] / ang, y = r[1] / ang, z = r[2] / ang;
    const double s = sin(ang), c = 1.0 - cos(ang);
    R[0] = 1.0 - c * (y * y + z * z); R[1] = c * (x * y) - s * z;       R[2] = c * (x * z) + s * y;
    R[3] = c * (x * y) + s * z;       R[4] = 1.0 - c * (x * x + z * z); R[5] = c * (y * z) - s * x;
    R[6] = c * (x * z) - s * y;       R[7] = c * (y * z) + s * x;       R[8] = 1.0 - c * (x * x + y * y);
}

// one row: pose [72] axis-angles, J [24][3] the rest joints of its shape, trans [3]; writes pf [207] and A [24][AROW] in fp32, and the posed
// joints [24][3] + trans in fp64 when joints is not null.  parents[0] = -1, parents[k] < k.
__device__ __forceinline__ void row_chain(const int *parents, const double *pose, const double *J, const double *trans, float *pf, float *A,
                                          double *joints) {
    double G[NJ][12];                  // rotation row-major, then the translation
    for (int k = 0; k < NJ; k++) {
        double R[9];
        rodrigues(pose + 3 * k, R);
        if (k > 0)
            for (int i = 0; i < 9; i++) pf[(k - 1) * 9 + i] = (float)(R[i] - ((i & 3) == 0 ? 1.0 : 0.0));
        double *g = G[k];
        if (k == 0) {
            for (int i = 0; i < 9; i++) g[i] = R[i];
            for (int i = 0; i < 3; i++) g[9 + i] = J[i];
        } else {
            const int p = parents[k];
            const double *P = G[p];
            const double t[3] = {J[3 * k] - J[3 * p], J[3 * k + 1] - J[3 * p + 1], J[3 * k + 2] - J[3 * p + 2]};
            for (int i = 0; i < 3; i++) {
                for (int c = 0; c < 3; c++) g[3 * i + c] = P[3 * i] * R[c] + P[3 * i + 1] * R[3 + c] + P[3 * i + 2] * R[6 + c];
                g[9 + i] = P[3 * i] * t[0] + P[3 * i + 1] * t[1] + P[3 * i + 2] * t[2] + P[9 + i];
            }
        }
        for (int i = 0; i < 3; i++) {
            const double gj = g[3 * i] * J[3 * k] + g[3 * i + 1] * J[3 * k + 1] + g[3 * i + 2] * J[3 * k + 2];
            for (int c = 0; c < 3; c++) A[AROW * k + 4 * i + c] = (float)g[3 * i + c];
            A[AROW * k + 4 * i + 3] = (float)(g[9 + i] - gj);
            if (joints) joints[3 * k + i] = g[9 + i] + trans[i];
        }
    }
}

}  // namespace meshm
}  // namespace uhc
