// curriculum.cu -- the failure-weighted curriculum after each rollout, on the device (curriculum_core.h; C ABI in step_kernel.cu).
// Compiled on its own with -fmad=false: the weights restate failure_weights' fp64 numpy arithmetic operation for operation.
//
// One update is four launches on the caller's stream and no host synchronise:
//   k_cur_rank     per block of UPD_CHUNK log entries: each ended episode's rank among the same clip's entries before it in the block,
//                  and the block's count per clip (the counts are sums, so atomics do not decide any order)
//   k_cur_scan     per clip: exclusive scan of the block counts (each entry's rank within its clip over the whole log) and the total
//   k_cur_scatter  every entry among the last max_freq of its clip goes to ring slot (head + rank) mod max_freq
//   k_cur_weights  one block: rings advance, s_c = ewma, p = exp(-s / temp), numpy's pairwise sum, w = freq * p / sum + (1 - freq) / C
//                  in fp32, and the CDF as a fixed-order fp64 scan, written in place into the sampler's CDF
// The global curriculum adds k_cur_stage (this rank's log into its slot of the payload the gradient all-reduce sums) and k_cur_unpack (the
// summed payload back into one [world T E] log, which the four launches above then take as any other log).
#include <cuda_runtime.h>
#include "curriculum_core.h"

namespace uhc {
namespace cur {

__global__ void __launch_bounds__(UPD_CHUNK) k_cur_rank(const int *__restrict__ clip_log, int N, int C, int *__restrict__ cnt, int *__restrict__ rank) {
    __shared__ int s_clip[UPD_CHUNK];
    const int i = blockIdx.x * UPD_CHUNK + threadIdx.x;
    int c = i < N ? clip_log[i] : -1;
    if (c >= C) c = -1;
    s_clip[threadIdx.x] = c;
    __syncthreads();
    if (c < 0) return;
    int r = 0;
    for (int j = 0; j < (int)threadIdx.x; j++) r += s_clip[j] == c;
    rank[i] = r;
    atomicAdd(cnt + (size_t)blockIdx.x * C + c, 1);
}

__global__ void k_cur_scan(int *__restrict__ cnt, int nchunk, int C, int *__restrict__ ncl) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    int run = 0;
    for (int b = 0; b < nchunk; b++) { const int v = cnt[(size_t)b * C + c]; cnt[(size_t)b * C + c] = run; run += v; }
    ncl[c] = run;
}

__global__ void k_cur_scatter(Dev d, const int *__restrict__ clip_log, const float *__restrict__ pct_log, const int *__restrict__ start_log, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int c = clip_log[i];
    if (c < 0 || c >= d.C) return;
    const int s = d.cnt[(size_t)(i / UPD_CHUNK) * d.C + c] + d.rank[i];
    if (!keep_rank(s, d.ncl[c], d.M)) return;
    const int slot = rank_slot(d.meta, d.M, c, s % d.M);
    d.pct[(size_t)c * d.M + slot] = pct_log[i]; d.start[(size_t)c * d.M + slot] = start_log[i];
}

constexpr int WT = 1024;
__global__ void __launch_bounds__(WT) k_cur_weights(Dev d, int advance) {
    __shared__ double s_sum, s_part[WT];
    const int C = d.C;
    int any = 0;
    for (int c = threadIdx.x; c < C; c += WT) {
        if (advance) ring_advance(d.meta, d.M, c, d.ncl[c]);
        any |= d.meta[2 * c + 1] > 0;
        d.p[c] = exp(-success_ewma(d.pct, d.meta, d.M, c) / d.temp);
    }
    any = __syncthreads_or(any);
    __threadfence_block();
    if (threadIdx.x == 0) s_sum = pairwise_sum(d.p, C);
    __syncthreads();
    // weights, then the CDF: contiguous runs per thread summed in order, a fixed tree over the runs (same order every call)
    const int per = (C + WT - 1) / WT, c0 = threadIdx.x * per, c1 = c0 + per < C ? c0 + per : C;
    double run = 0.0;
    for (int c = c0; c < c1; c++) {
        const float w = any ? clip_weight(d.p[c], s_sum, d.freq, C)
                            : (float)(d.t_max > 0 ? (d.clip_adr[c + 1] - d.clip_adr[c]) / d.t_max + 1 : 1);   // sample_keys rule
        d.p[c] = (double)w;
        run += (double)w;
    }
    s_part[threadIdx.x] = run;
    __syncthreads();
    for (int off = 1; off < WT; off <<= 1) {          // inclusive Hillis-Steele scan of the run sums
        const double v = threadIdx.x >= (unsigned)off ? s_part[threadIdx.x - off] : 0.0;
        __syncthreads();
        s_part[threadIdx.x] += v;
        __syncthreads();
    }
    double acc = threadIdx.x > 0 ? s_part[threadIdx.x - 1] : 0.0;
    for (int c = c0; c < c1; c++) { acc += d.p[c]; d.cdf[c] = (float)acc; }
}

cudaError_t launch_update(const Dev &d, const int *clip_log, const float *pct_log, const int *start_log, int N, cudaStream_t st) {
    const int nchunk = (N + UPD_CHUNK - 1) / UPD_CHUNK;
    cudaError_t ce = cudaMemsetAsync(d.cnt, 0, (size_t)nchunk * d.C * sizeof(int), st);
    if (ce != cudaSuccess) return ce;
    k_cur_rank<<<nchunk, UPD_CHUNK, 0, st>>>(clip_log, N, d.C, d.cnt, d.rank);
    k_cur_scan<<<(d.C + 255) / 256, 256, 0, st>>>(d.cnt, nchunk, d.C, d.ncl);
    k_cur_scatter<<<(N + 255) / 256, 256, 0, st>>>(d, clip_log, pct_log, start_log, N);
    k_cur_weights<<<1, WT, 0, st>>>(d, 1);
    return cudaGetLastError();
}

cudaError_t launch_weights(const Dev &d, cudaStream_t st) {
    k_cur_weights<<<1, WT, 0, st>>>(d, 0);
    return cudaGetLastError();
}

__global__ void k_cur_stage(const int *__restrict__ clip_log, const float *__restrict__ pct_log, const int *__restrict__ start_log, int n, float *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) stage_entry(clip_log[i], pct_log[i], start_log[i], out + 3 * (size_t)i);
}

__global__ void k_cur_unpack(const float *__restrict__ in, int n, int *__restrict__ clip_log, float *__restrict__ pct_log, int *__restrict__ start_log) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) unpack_entry(in + 3 * (size_t)i, clip_log + i, pct_log + i, start_log + i);
}

cudaError_t launch_stage(const int *clip_log, const float *pct_log, const int *start_log, int n, float *out, cudaStream_t st) {
    k_cur_stage<<<(n + 255) / 256, 256, 0, st>>>(clip_log, pct_log, start_log, n, out);
    return cudaGetLastError();
}

cudaError_t launch_unpack(const float *in, int n, int *clip_log, float *pct_log, int *start_log, cudaStream_t st) {
    k_cur_unpack<<<(n + 255) / 256, 256, 0, st>>>(in, n, clip_log, pct_log, start_log);
    return cudaGetLastError();
}

}  // namespace cur
}  // namespace uhc
