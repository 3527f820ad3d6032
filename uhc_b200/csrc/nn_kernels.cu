// nn_kernels.cu -- policy / value MLP, Gaussian head, observation normaliser, GAE and the PPO update as hand-written
// CUDA kernels behind the C ABI (include/uhc_nn.h).  Reference rows (SURVEY.md section 8a):
//   a12 ZFilter            uhc/khrylib/utils/zfilter.py:7-73
//   a13 PolicyGaussian     uhc/khrylib/rl/core/policy_gaussian.py:26-31, models/mlp.py:24-27, core/distributions.py:6-25
//   a14 Value              uhc/khrylib/rl/core/critic.py:15-18
//   a15 estimate_advantages uhc/khrylib/rl/core/common.py:5-25
//   a16 update_policy/ppo_loss/update_value/clip grad  uhc/khrylib/rl/agents/agent_ppo.py:16-65, agent_pg.py:18-25; torch.optim.Adam
// This file holds the fp32 SIMT GEMM (all three layouts) and every streaming kernel; the wgmma tensor-core GEMM used
// for the rollout-time forward lives in mlp_wgmma.cu.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string>
#include "../../include/uhc_nn.h"
#include "errors.h"

// ------------------------------------------------------------------------------------------------ activations
__device__ __forceinline__ float act_fwd(float z, int act) {
    switch (act) {
    case UHC_ACT_GELU: return 0.5f * z * (1.0f + erff(z * 0.70710678118654752f));
    case UHC_ACT_TANH: return tanhf(z);
    case UHC_ACT_RELU: return z > 0.f ? z : 0.f;
    case UHC_ACT_SIGMOID: return 1.0f / (1.0f + expf(-z));
    }
    return z;
}
__device__ __forceinline__ float act_bwd(float z, int act) {
    switch (act) {
    case UHC_ACT_GELU: return 0.5f * (1.0f + erff(z * 0.70710678118654752f)) + z * 0.3989422804014327f * expf(-0.5f * z * z);
    case UHC_ACT_TANH: { float t = tanhf(z); return 1.0f - t * t; }
    case UHC_ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case UHC_ACT_SIGMOID: { float s = 1.0f / (1.0f + expf(-z)); return s * (1.0f - s); }
    }
    return 1.f;
}

// ------------------------------------------------------------------------------------------------ SIMT GEMM
// C[i][j] = epilogue( sum_r A(i,r) * B(r,j) ),  i < M, j < N, r < R, with arbitrary element strides:
//   A(i,r) = A[i*sai + r*sar],  B(r,j) = B[r*sbr + j*sbj].  128x128x16 tiles, 256 threads, 8x8 outputs per thread.
// Epilogue: + bias[j], optional pre-activation store Z, activation, optional accumulate into C (beta = 1).
template <bool A_R_CONTIG, bool B_J_CONTIG>
__global__ void __launch_bounds__(256)
k_gemm(const float *__restrict__ A, const float *__restrict__ B, float *__restrict__ C, float *__restrict__ Z, const float *__restrict__ bias,
       int M, int N, int R, long sai, long sar, long sbr, long sbj, int act, int accumulate) {
    constexpr int BM = 128, BN = 128, BK = 16;
    __shared__ float As[BK][BM + 4], Bs[BK][BN + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
    float acc[8][8];
#pragma unroll
    for (int a = 0; a < 8; a++)
#pragma unroll
        for (int b = 0; b < 8; b++) acc[a][b] = 0.f;
    for (int r0 = 0; r0 < R; r0 += BK) {
#pragma unroll
        for (int l = 0; l < 8; l++) {  // 2048 elements per tile / 256 threads
            const int e = tid + 256 * l;
            int ii, rr;
            if (A_R_CONTIG) { rr = e & 15; ii = e >> 4; } else { ii = e & 127; rr = e >> 7; }
            const int gi = i0 + ii, gr = r0 + rr;
            As[rr][ii] = (gi < M && gr < R) ? A[gi * sai + gr * sar] : 0.f;
            int jj, r2;
            if (B_J_CONTIG) { jj = e & 127; r2 = e >> 7; } else { r2 = e & 15; jj = e >> 4; }
            const int gj = j0 + jj, gr2 = r0 + r2;
            Bs[r2][jj] = (gj < N && gr2 < R) ? B[gr2 * sbr + gj * sbj] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; k++) {
            float a[8], b[8];
#pragma unroll
            for (int u = 0; u < 8; u++) { a[u] = As[k][ty * 8 + u]; b[u] = Bs[k][tx * 8 + u]; }
#pragma unroll
            for (int u = 0; u < 8; u++)
#pragma unroll
                for (int v = 0; v < 8; v++) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int gi = i0 + ty * 8 + u;
        if (gi >= M) continue;
#pragma unroll
        for (int v = 0; v < 8; v++) {
            const int gj = j0 + tx * 8 + v;
            if (gj >= N) continue;
            float z = acc[u][v] + (bias ? bias[gj] : 0.f);
            const size_t o = (size_t)gi * N + gj;
            if (accumulate) z += C[o];
            if (Z) Z[o] = z;
            C[o] = act_fwd(z, act);
        }
    }
}

static int launch_gemm(const float *A, const float *B, float *C, float *Z, const float *bias, int M, int N, int R, long sai, long sar,
                       long sbr, long sbj, int act, int accumulate, cudaStream_t st) {
    dim3 grid((N + 127) / 128, (M + 127) / 128);
    const bool ar = (sar == 1), bj = (sbj == 1);
    if (ar && bj) k_gemm<true, true><<<grid, 256, 0, st>>>(A, B, C, Z, bias, M, N, R, sai, sar, sbr, sbj, act, accumulate);
    else if (ar && !bj) k_gemm<true, false><<<grid, 256, 0, st>>>(A, B, C, Z, bias, M, N, R, sai, sar, sbr, sbj, act, accumulate);
    else if (!ar && bj) k_gemm<false, true><<<grid, 256, 0, st>>>(A, B, C, Z, bias, M, N, R, sai, sar, sbr, sbj, act, accumulate);
    else k_gemm<false, false><<<grid, 256, 0, st>>>(A, B, C, Z, bias, M, N, R, sai, sar, sbr, sbj, act, accumulate);
    CK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ streaming kernels
// dz = dh * act'(z)  (in place on dh allowed)
__global__ void k_act_bwd(const float *__restrict__ dh, const float *__restrict__ z, float *__restrict__ dz, size_t n, int act) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dz[i] = dh[i] * act_bwd(z[i], act);
}
// column sums: out[j] = sum_i X[i][j]   (bias gradients), one block per 32 columns
__global__ void k_colsum(const float *__restrict__ X, float *__restrict__ out, int M, int N) {
    __shared__ float red[32][33];
    const int j = blockIdx.x * 32 + threadIdx.x;
    float s = 0.f;
    if (j < N) for (int i = threadIdx.y; i < M; i += blockDim.y) s += X[(size_t)i * N + j];
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && j < N) { float t = 0.f; for (int k = 0; k < 32; k++) t += red[k][threadIdx.x]; out[j] = t; }
}

// counter-based RNG (philox-style mixing is overkill here: splitmix64 per (seed, stream, index) + Box-Muller).
// u1 = (k + 1) * fp32(1 / (2^24 + 2)), k < 2^24, lies in (0, 1): the scale is spelled as its exact fp32 value, the one the earlier
// literal 1.0f / 16777217.0f compiled to, so the stream of normals is unchanged and a host restatement can reproduce it bit for bit.
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}
__device__ __forceinline__ float gauss_from(uint64_t seed, uint64_t idx) {
    const uint64_t h = splitmix64(seed ^ splitmix64(idx));
    const float u1 = ((uint32_t)(h >> 40) + 1.0f) * 0x1.fffffcp-25f, u2 = (uint32_t)(h & 0xFFFFFF) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
// a = mean + exp(log_std) * eps (or mean when mean_action[i] != 0); logp = sum_d Normal(mean, std).log_prob(a)
// (policy.py:12-15 select_action, distributions.py:21-22).  One warp per row.
__global__ void k_gauss_sample(const float *__restrict__ mean, const float *__restrict__ log_std, const uint8_t *__restrict__ mean_action,
                               float *__restrict__ action, float *__restrict__ logp, int M, int A, uint64_t seed, uint64_t step) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    const bool det = mean_action && mean_action[row];
    float lp = 0.f;
    for (int d = lane; d < A; d += 32) {
        const float mu = mean[(size_t)row * A + d], ls = log_std[d], sd = expf(ls);
        const float eps = det ? 0.f : gauss_from(seed, (step * (uint64_t)M + row) * (uint64_t)A + d);
        const float a = mu + sd * eps;
        action[(size_t)row * A + d] = a;
        const float zq = (a - mu) / sd;
        lp += -0.5f * zq * zq - ls - 0.91893853320467274178f;
    }
    for (int o = 16; o; o >>= 1) lp += __shfl_xor_sync(0xffffffffu, lp, o);
    if (lane == 0 && logp) logp[row] = lp;
}
__global__ void k_gauss_logprob(const float *__restrict__ mean, const float *__restrict__ log_std, const float *__restrict__ action,
                                float *__restrict__ logp, int M, int A) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    float lp = 0.f;
    for (int d = lane; d < A; d += 32) {
        const float mu = mean[(size_t)row * A + d], ls = log_std[d], zq = (action[(size_t)row * A + d] - mu) * expf(-ls);
        lp += -0.5f * zq * zq - ls - 0.91893853320467274178f;
    }
    for (int o = 16; o; o >>= 1) lp += __shfl_xor_sync(0xffffffffu, lp, o);
    if (lane == 0) logp[row] = lp;
}

// PPO clipped surrogate (agent_ppo.py:58-65) over rows with exps != 0:  L = -mean_i min(r A, clip(r,1-e,1+e) A), r = exp(logp - fixed).
// Writes dL/dmean [M][A] (zero rows where exps == 0) and accumulates the loss and the selected-row count.
__global__ void k_ppo_grad(const float *__restrict__ mean, const float *__restrict__ log_std, const float *__restrict__ action,
                           const float *__restrict__ adv, const float *__restrict__ fixed_logp, const float *__restrict__ exps, float clip_eps,
                           float inv_count, float *__restrict__ dmean, float *__restrict__ loss_acc, int M, int A, const float *__restrict__ inv_count_dev) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    if (inv_count_dev) inv_count = *inv_count_dev;   // 1 / #selected rows of the GLOBAL batch, produced on the device (multi-GPU: after the all-reduce)
    const bool sel = exps[row] != 0.f;
    float lp = 0.f;
    for (int d = lane; d < A; d += 32) {
        const float mu = mean[(size_t)row * A + d], ls = log_std[d], zq = (action[(size_t)row * A + d] - mu) * expf(-ls);
        lp += -0.5f * zq * zq - ls - 0.91893853320467274178f;
    }
    for (int o = 16; o; o >>= 1) lp += __shfl_xor_sync(0xffffffffu, lp, o);
    const float ratio = expf(lp - fixed_logp[row]), a = adv[row];
    const float s1 = ratio * a, s2 = fminf(fmaxf(ratio, 1.f - clip_eps), 1.f + clip_eps) * a;
    // d(-min(s1,s2))/dlogp: -ratio*a when the unclipped branch is the minimum (ties -> torch.min takes surr1's gradient path equally; use <=)
    const float g = (sel && s1 <= s2) ? -ratio * a * inv_count : 0.f;
    for (int d = lane; d < A; d += 32) {
        const float mu = mean[(size_t)row * A + d], ls = log_std[d];
        dmean[(size_t)row * A + d] = g * (action[(size_t)row * A + d] - mu) * expf(-2.f * ls);
    }
    if (lane == 0 && sel && loss_acc) atomicAdd(loss_acc, -fminf(s1, s2) * inv_count);
}
// value loss (agent_pg.py:18-25): L = mean (v - ret)^2 ; dv = 2 (v - ret) / M
__global__ void k_value_grad(const float *__restrict__ v, const float *__restrict__ ret, float *__restrict__ dv, float *__restrict__ loss_acc, int M, float Mtot) {
    float s = 0.f;   // Mtot: rows of the GLOBAL batch (= M on one GPU): the gradients of the shards then SUM to the full-batch mean gradient
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x) { const float d = v[i] - ret[i]; dv[i] = 2.f * d / Mtot; s += d * d / Mtot; }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0 && loss_acc) atomicAdd(loss_acc, s);
}
// sum of squares (gradient norm), double accumulation
__global__ void k_sqsum(const float *__restrict__ x, size_t n, double *__restrict__ out) {
    double s = 0.0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) s += (double)x[i] * x[i];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, s);
}
// Adam (torch.optim.Adam defaults: no weight decay, no amsgrad) with an optional global-norm clip factor read from the device:
// scale = min(1, max_norm / (sqrt(*sqnorm) + 1e-6))  (torch.nn.utils.clip_grad_norm_, agent_ppo.py:53-56)
__global__ void k_adam(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v, size_t n, float lr,
                       float b1, float b2, float eps, float bc1, float bc2, const double *__restrict__ sqnorm, float max_norm) {
    float scale = 1.f;
    if (sqnorm) { const float nrm = (float)sqrt(*sqnorm); const float c = max_norm / (nrm + 1e-6f); scale = c < 1.f ? c : 1.f; }
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float gi = g[i] * scale;
        const float mi = b1 * m[i] + (1.f - b1) * gi, vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi; v[i] = vi;
        p[i] -= lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
    }
}

// GAE over a [T][E] rollout (time-major): one thread per env, reverse scan (common.py:5-25 semantics per trajectory):
//   delta = r + gamma * V' * mask - V ; A = delta + gamma * tau * A' * mask ; V' = next value (bootstrap `last_value` at t = T-1,
//   which the reference never needs because it only collects whole episodes -- SURVEY.md Appendix C).  returns = V + A.
__global__ void k_gae(const float *__restrict__ rew, const float *__restrict__ mask, const float *__restrict__ val, const float *__restrict__ last_val,
                      float gamma, float tau, float *__restrict__ adv, float *__restrict__ ret, int T, int E) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    float pv = last_val ? last_val[e] : 0.f, pa = 0.f;
    for (int t = T - 1; t >= 0; --t) {
        const size_t i = (size_t)t * E + e;
        const float mk = mask[i], v = val[i];
        const float delta = rew[i] + gamma * pv * mk - v;
        const float a = delta + gamma * tau * pa * mk;
        adv[i] = a; ret[i] = v + a;
        pv = v; pa = a;
    }
}
// sum and sum of squares in double (advantage normalisation: (A - mean) / std_unbiased, common.py:22)
__global__ void k_moments(const float *__restrict__ x, size_t n, double *__restrict__ out2) {
    double s = 0.0, q = 0.0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) { const double v = x[i]; s += v; q += v * v; }
    for (int o = 16; o; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
    if ((threadIdx.x & 31) == 0) { atomicAdd(out2, s); atomicAdd(out2 + 1, q); }
}
__global__ void k_normalize(float *__restrict__ x, size_t n, const double *__restrict__ mom, const double *__restrict__ ntot_dev) {
    const double N = ntot_dev ? *ntot_dev : (double)n;    // elements behind the moments (the global batch when they were all-reduced)
    const double mean = mom[0] / N, var = (mom[1] - N * mean * mean) / (N - 1.0);
    const float mu = (float)mean, inv = (float)(1.0 / sqrt(var));
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) x[i] = (x[i] - mu) * inv;
}

// ZFilter (zfilter.py:7-73): running mean / var over every observation seen, y = clip((x - mean) / (std + 1e-8), -clip, clip).
// Batched form: Chan et al. merge of the batch moments into the running (n, mean, S) state, then normalise the batch with the
// UPDATED statistics (the reference pushes then normalises each sample; sequential-vs-batched order is the documented deviation).
// stats layout: [0] = n (as double), then mean[D], S[D] (doubles).  One block per 32 dims (column reduction).
constexpr int ZF_CHUNKS = 16;   // row chunks of the batch-moment pass (deterministic two-stage reduction: partials, then a fixed-order merge)
// A column that holds one value in every row of the batch (the shape vector while every env holds one subject) is detected exactly: stage 1 also
// counts the rows that differ from the batch's first row.  Such a column takes that value as its batch mean and 0 as its spread; from raw sums,
// S2 - n mean^2 leaves a rounding residue of either sign there, and a negative S normalised the column to NaN -> -clip.  Every other column keeps
// the raw-sum arithmetic, clamped at 0, so the statistics of a batch without such a residue are unchanged to the last bit.
// stage 1: block (column tile, row chunk) -> partial (sum, sum of squares, rows != first row) of its rows for 32 columns, into ws[chunk][D][3]
__global__ void k_zfilter_partial(const float *__restrict__ X, int M, int D, double *__restrict__ ws) {
    __shared__ double rs[32][33], rq[32][33];
    __shared__ int rd[32][33];
    const int j = blockIdx.x * 32 + threadIdx.x, ch = blockIdx.y;
    const int r0 = (int)(((long)M * ch) / ZF_CHUNKS), r1 = (int)(((long)M * (ch + 1)) / ZF_CHUNKS);
    double s = 0.0, q = 0.0;
    int nd = 0;
    if (j < D) {
        const float c = X[j];
        for (int i = r0 + threadIdx.y; i < r1; i += blockDim.y) { const float x = X[(size_t)i * D + j]; const double v = x; s += v; q += v * v; nd += x != c; }
    }
    rs[threadIdx.y][threadIdx.x] = s; rq[threadIdx.y][threadIdx.x] = q; rd[threadIdx.y][threadIdx.x] = nd;
    __syncthreads();
    if (threadIdx.y == 0 && j < D) {
        double S1 = 0.0, S2 = 0.0;
        int N = 0;
        for (int k = 0; k < 32; k++) { S1 += rs[k][threadIdx.x]; S2 += rq[k][threadIdx.x]; N += rd[k][threadIdx.x]; }
        double *w = ws + ((size_t)ch * D + j) * 3;
        w[0] = S1; w[1] = S2; w[2] = (double)N;
    }
}
// stage 2: fixed-order sum of the chunk partials, Chan merge into the running (n, mean, S); k_zfilter_count bumps the count after it
__global__ void k_zfilter_merge(const float *__restrict__ X, int M, int D, double *__restrict__ stats, const double *__restrict__ ws) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= D) return;
    double S1 = 0.0, S2 = 0.0, nd = 0.0;
    for (int ch = 0; ch < ZF_CHUNKS; ch++) { const double *w = ws + ((size_t)ch * D + j) * 3; S1 += w[0]; S2 += w[1]; nd += w[2]; }
    const bool constant = nd == 0.0;
    const double nb = (double)M, mb = constant ? (double)X[j] : S1 / nb, Sb = constant ? 0.0 : fmax(0.0, S2 - nb * mb * mb);
    const double na = stats[0], ma = stats[1 + j], Sa = stats[1 + D + j];
    const double n = na + nb, dlt = mb - ma;
    stats[1 + j] = ma + dlt * nb / n;              // from empty statistics: c nb is exact (c fp32, nb < 2^29), so a constant column's mean is c
    stats[1 + D + j] = fmax(0.0, Sa + Sb + dlt * dlt * na * nb / n);
}
__global__ void k_zfilter_count(double *stats, int M) { stats[0] += (double)M; }
__global__ void k_zfilter_apply(const float *__restrict__ X, float *__restrict__ Y, int M, int D, const double *__restrict__ stats, float clip) {
    const double n = stats[0];
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)M * D; i += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % D);
        const double mean = stats[1 + j], var = n > 1.0 ? stats[1 + D + j] / (n - 1.0) : mean * mean;
        float y = (float)(((double)X[i] - mean) / (sqrt(var) + 1e-8));
        if (clip > 0.f) y = fminf(fmaxf(y, -clip), clip);
        Y[i] = y;
    }
}

// ------------------------------------------------------------------------------------------------ C ABI
// ---- PolicyMCP (uhc/models/policy_mcp.py:28-36): action_mean = sum_k softmax(composer(x))_k * primitive_k(x).  One warp per row.
// xall = [P][M][A] primitive outputs, c = [M][P] composer outputs (after its last activation), weight = softmax(c) kept for the backward pass.
constexpr int MCP_MAX_PRIM = 16;
__global__ void __launch_bounds__(256) k_mcp_combine(const float *__restrict__ xall, const float *__restrict__ c, float *__restrict__ weight, float *__restrict__ mean,
                                                     int M, int A, int P) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    float w[MCP_MAX_PRIM]; float mx = -3.0e38f, den = 0.f;
    for (int k = 0; k < P; k++) { w[k] = c[(size_t)row * P + k]; mx = fmaxf(mx, w[k]); }
    for (int k = 0; k < P; k++) { w[k] = expf(w[k] - mx); den += w[k]; }
    const float inv = 1.0f / den;
    for (int k = 0; k < P; k++) { w[k] *= inv; if (weight && lane == 0) weight[(size_t)row * P + k] = w[k]; }
    for (int a = lane; a < A; a += 32) {
        float s = 0.f;
        for (int k = 0; k < P; k++) s += w[k] * xall[((size_t)k * M + row) * A + a];
        mean[(size_t)row * A + a] = s;
    }
}
// d xall_k = w_k dmean ; d w_k = sum_a dmean_a xall_k,a ; softmax backward d c_k = w_k (d w_k - sum_j w_j d w_j)
__global__ void __launch_bounds__(256) k_mcp_backward(const float *__restrict__ xall, const float *__restrict__ weight, const float *__restrict__ dmean,
                                                      float *__restrict__ dxall, float *__restrict__ dc, int M, int A, int P) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    float w[MCP_MAX_PRIM], dw[MCP_MAX_PRIM];
    for (int k = 0; k < P; k++) { w[k] = weight[(size_t)row * P + k]; dw[k] = 0.f; }
    for (int a = lane; a < A; a += 32) {
        const float g = dmean[(size_t)row * A + a];
        for (int k = 0; k < P; k++) {
            const size_t i = ((size_t)k * M + row) * A + a;
            dw[k] += g * xall[i];
            dxall[i] = w[k] * g;
        }
    }
    float dot = 0.f;
    for (int k = 0; k < P; k++) { for (int o = 16; o; o >>= 1) dw[k] += __shfl_xor_sync(0xffffffffu, dw[k], o); dot += w[k] * dw[k]; }
    if (lane == 0) for (int k = 0; k < P; k++) dc[(size_t)row * P + k] = w[k] * (dw[k] - dot);
}

extern "C" {
int uhc_linear_forward(const float *x, const float *W, const float *b, float *y, float *z_or_null, int M, int N, int K, int act, void *stream) {
    return launch_gemm(x, W, y, z_or_null, b, M, N, K, K, 1, 1, K, act, 0, (cudaStream_t)stream);   // y = act(x W^T + b)
}
int uhc_linear_backward(const float *x, const float *W, const float *dz, float *dx_or_null, float *dW, float *db, int M, int N, int K, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (dx_or_null && launch_gemm(dz, W, dx_or_null, nullptr, nullptr, M, K, N, N, 1, K, 1, UHC_ACT_NONE, 0, st)) return -1;   // dx = dz W
    if (launch_gemm(dz, x, dW, nullptr, nullptr, N, K, M, 1, N, K, 1, UHC_ACT_NONE, 0, st)) return -1;                           // dW = dz^T x
    if (db) { k_colsum<<<(N + 31) / 32, dim3(32, 32), 0, st>>>(dz, db, M, N); CK(cudaGetLastError()); }
    return 0;
}
int uhc_act_backward(const float *dh, const float *z, float *dz, long n, int act, void *stream) {
    k_act_bwd<<<1056, 256, 0, (cudaStream_t)stream>>>(dh, z, dz, (size_t)n, act); CK(cudaGetLastError()); return 0;
}
int uhc_gaussian_sample(const float *mean, const float *log_std, const unsigned char *mean_action, float *action, float *logp, int M, int A,
                        unsigned long long seed, unsigned long long step, void *stream) {
    k_gauss_sample<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>(mean, log_std, mean_action, action, logp, M, A, seed, step); CK(cudaGetLastError()); return 0;
}
int uhc_gaussian_logprob(const float *mean, const float *log_std, const float *action, float *logp, int M, int A, void *stream) {
    k_gauss_logprob<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>(mean, log_std, action, logp, M, A); CK(cudaGetLastError()); return 0;
}
int uhc_ppo_policy_grad(const float *mean, const float *log_std, const float *action, const float *adv, const float *fixed_logp, const float *exps,
                        float clip_eps, float inv_count, float *dmean, float *loss_acc, int M, int A, void *stream) {
    k_ppo_grad<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>(mean, log_std, action, adv, fixed_logp, exps, clip_eps, inv_count, dmean, loss_acc, M, A, nullptr);
    CK(cudaGetLastError()); return 0;
}
int uhc_ppo_policy_grad_dev(const float *mean, const float *log_std, const float *action, const float *adv, const float *fixed_logp, const float *exps,
                            float clip_eps, const float *inv_count_dev, float *dmean, float *loss_acc, int M, int A, void *stream) {
    if (!inv_count_dev) { uhc_err() = "uhc_ppo_policy_grad_dev: inv_count_dev is null"; return -2; }
    k_ppo_grad<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>(mean, log_std, action, adv, fixed_logp, exps, clip_eps, 0.f, dmean, loss_acc, M, A, inv_count_dev);
    CK(cudaGetLastError()); return 0;
}
int uhc_value_grad(const float *v, const float *ret, float *dv, float *loss_acc, int M, void *stream) {
    k_value_grad<<<592, 256, 0, (cudaStream_t)stream>>>(v, ret, dv, loss_acc, M, (float)M); CK(cudaGetLastError()); return 0;
}
int uhc_value_grad_n(const float *v, const float *ret, float *dv, float *loss_acc, int M, long M_total, void *stream) {
    k_value_grad<<<592, 256, 0, (cudaStream_t)stream>>>(v, ret, dv, loss_acc, M, (float)M_total); CK(cudaGetLastError()); return 0;
}
int uhc_sqsum(const float *x, long n, double *out_acc, void *stream) {
    k_sqsum<<<592, 256, 0, (cudaStream_t)stream>>>(x, (size_t)n, out_acc); CK(cudaGetLastError()); return 0;
}
int uhc_adam_step(float *p, const float *g, float *m, float *v, long n, float lr, float beta1, float beta2, float eps, int step,
                  const double *sqnorm_or_null, float max_norm, void *stream) {
    const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
    k_adam<<<1056, 256, 0, (cudaStream_t)stream>>>(p, g, m, v, (size_t)n, lr, beta1, beta2, eps, bc1, bc2, sqnorm_or_null, max_norm);
    CK(cudaGetLastError()); return 0;
}
int uhc_gae(const float *rew, const float *mask, const float *val, const float *last_val, float gamma, float tau, float *adv, float *ret, int T, int E,
            void *stream) {
    k_gae<<<(E + 127) / 128, 128, 0, (cudaStream_t)stream>>>(rew, mask, val, last_val, gamma, tau, adv, ret, T, E); CK(cudaGetLastError()); return 0;
}
int uhc_normalize_advantages(float *adv, long n, double *scratch2, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemsetAsync(scratch2, 0, 2 * sizeof(double), st));
    k_moments<<<592, 256, 0, st>>>(adv, (size_t)n, scratch2); CK(cudaGetLastError());
    k_normalize<<<592, 256, 0, st>>>(adv, (size_t)n, scratch2, nullptr); CK(cudaGetLastError());
    return 0;
}
// the two halves of the same normalisation, for a batch sharded over GPUs: local (sum, sum of squares) -> [all-reduce] -> normalise with
// the global moments and the global element count (both read from device memory: no host round trip between the collective and the kernel)
int uhc_adv_moments(const float *adv, long n, double *out2, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemsetAsync(out2, 0, 2 * sizeof(double), st));
    k_moments<<<592, 256, 0, st>>>(adv, (size_t)n, out2); CK(cudaGetLastError());
    return 0;
}
int uhc_adv_normalize(float *adv, long n, const double *mom2_dev, const double *ntotal_dev, void *stream) {
    k_normalize<<<592, 256, 0, (cudaStream_t)stream>>>(adv, (size_t)n, mom2_dev, ntotal_dev); CK(cudaGetLastError());
    return 0;
}
int uhc_mcp_combine(const float *xall, const float *c, float *weight_or_null, float *mean, int M, int A, int P, void *stream) {
    if (P < 1 || P > MCP_MAX_PRIM) { uhc_err() = "uhc_mcp_combine: 1..16 primitives"; return -2; }
    k_mcp_combine<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>(xall, c, weight_or_null, mean, M, A, P); CK(cudaGetLastError()); return 0;
}
int uhc_mcp_backward(const float *xall, const float *weight, const float *dmean, float *dxall, float *dc, int M, int A, int P, void *stream) {
    if (P < 1 || P > MCP_MAX_PRIM) { uhc_err() = "uhc_mcp_backward: 1..16 primitives"; return -2; }
    k_mcp_backward<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>(xall, weight, dmean, dxall, dc, M, A, P); CK(cudaGetLastError()); return 0;
}
int uhc_zfilter_workspace_doubles(int D) { return ZF_CHUNKS * D * 3; }
int uhc_zfilter(const float *x, float *y, int M, int D, double *stats, float clip, int update, void *stream) {
    // without a caller workspace: one per (thread, D), allocated on first use (not legal inside a stream capture -- the rollout passes its own)
    static thread_local double *ws = nullptr; static thread_local int ws_d = 0, ws_dev = -1;
    int dev = 0; cudaGetDevice(&dev);
    if (update && (!ws || ws_d < D || ws_dev != dev)) { if (ws && ws_dev == dev) cudaFree(ws); CK(cudaMalloc((void **)&ws, (size_t)uhc_zfilter_workspace_doubles(D) * sizeof(double))); ws_d = D; ws_dev = dev; }
    return uhc_zfilter_ws(x, y, M, D, stats, clip, update, ws, stream);
}
int uhc_zfilter_ws(const float *x, float *y, int M, int D, double *stats, float clip, int update, double *workspace, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (M < 0 || D <= 0) { uhc_err() = "uhc_zfilter_ws: M >= 0 and D > 0"; return -2; }
    if (update && M > 0) {     // an empty batch leaves the statistics as they are
        if (!workspace) { uhc_err() = "uhc_zfilter_ws: workspace is null"; return -2; }
        k_zfilter_partial<<<dim3((D + 31) / 32, ZF_CHUNKS), dim3(32, 32), 0, st>>>(x, M, D, workspace); CK(cudaGetLastError());
        k_zfilter_merge<<<(D + 127) / 128, 128, 0, st>>>(x, M, D, stats, workspace); CK(cudaGetLastError());
        k_zfilter_count<<<1, 1, 0, st>>>(stats, M); CK(cudaGetLastError());
    }
    if (y) { k_zfilter_apply<<<592, 256, 0, st>>>(x, y, M, D, stats, clip); CK(cudaGetLastError()); }
    return 0;
}
}  // extern "C"
