// curriculum_core.h -- the failure-weighted curriculum of the training loop: per-clip outcome history, clip weights and the
// precision-mode start, in one place.
//
// Restates the reference's rules (the training loop's freq_dict):
//   history   agent_copycat.py:561,590-603: every ended episode appends [percent, fr_start] to its clip's list, in the order the
//             rollout produced them (step-major, env-minor here); after the whole rollout every list keeps its last max_freq entries.
//   weights   dataset_amass_single.py:183-186 + math_utils.py:25-29: s_c = ewma(hist_c[:, 0] == 1) (0 for an empty history),
//             p = exp(-s / temp) / sum(p), w = freq * p + (1 - freq) / C (uhc_b200/agent.py failure_weights), rounded to fp32.
//   start     dataset_amass_single.py:222-232 (precision_mode): with probability prec_freq, and only when the clip's history holds an
//             entry with percent != 1, one such entry is picked uniformly and start ~ U{max(idx - 20 - t_min, 0) .. min(idx + 20, L - t_min) - 1};
//             otherwise start ~ U{0 .. L - t_min - 1}.
// The history of clip c is a ring of M = max_freq (percent, start) slots: meta[2c] = the slot the next entry goes to, meta[2c + 1] = the
// number of valid entries (the oldest at slot head - len mod M).  The same source compiles as CUDA code (curriculum.cu with -fmad=false,
// and the sampler in env_step.h) and, with -DUHC_EMU, as host code for the CPU tests (-ffp-contract=off).
#pragma once
#include <math.h>

#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_CDEV __host__ __device__ __forceinline__
#define UHC_CDEV_REC static __host__ __device__
#else
#define UHC_CDEV static inline
#define UHC_CDEV_REC static
#endif

namespace uhc {
namespace cur {

constexpr double EWMA_ALPHA = 0.05;   // math_utils.py:25
constexpr int PREC_WINDOW = 20;       // dataset_amass_single.py:227-228
constexpr int MAX_FREQ_CAP = 4096;    // largest ring the C ABI accepts

UHC_CDEV int ring_slot(const int *meta, int M, int c, int k) {   // slot of the k-th oldest entry of clip c
    const int head = meta[2 * c], len = meta[2 * c + 1];
    return ((head - len + k) % M + M) % M;
}
UHC_CDEV void ring_push(float *pct, int *start, int *meta, int M, int c, float p, int s) {
    const int head = meta[2 * c];
    pct[(size_t)c * M + head] = p; start[(size_t)c * M + head] = s;
    meta[2 * c] = (head + 1) % M;
    if (meta[2 * c + 1] < M) meta[2 * c + 1]++;
}

// one rollout's entries of clip c (n of them, ranked s = 0 .. n - 1 in log order) land at once: rank s is kept iff it is among the
// last M, at slot (head + s) mod M; then the ring advances by n.  Same result as n ring_push calls in rank order.
UHC_CDEV bool keep_rank(int s, int n, int M) { return s >= n - M; }
UHC_CDEV int rank_slot(const int *meta, int M, int c, int s) { return (meta[2 * c] + s) % M; }
UHC_CDEV void ring_advance(int *meta, int M, int c, int n) {
    meta[2 * c] = (int)(((long long)meta[2 * c] + n) % M);
    meta[2 * c + 1] = meta[2 * c + 1] + n < M ? meta[2 * c + 1] + n : M;
}

// ewma of the success flags (percent == 1) in history order, fp64; 0 for an empty history
UHC_CDEV double success_ewma(const float *pct, const int *meta, int M, int c) {
    const int len = meta[2 * c + 1];
    if (len == 0) return 0.0;
    double avg = pct[(size_t)c * M + ring_slot(meta, M, c, 0)] == 1.0f ? 1.0 : 0.0;
    for (int k = 1; k < len; k++) {
        const double x = pct[(size_t)c * M + ring_slot(meta, M, c, k)] == 1.0f ? 1.0 : 0.0;
        avg = EWMA_ALPHA * x + (1.0 - EWMA_ALPHA) * avg;
    }
    return avg;
}

// numpy's pairwise summation of a contiguous float64 array (p.sum() in failure_weights), in its association order
UHC_CDEV_REC double pairwise_sum(const double *a, int n) {
    if (n < 8) { double res = 0.0; for (int i = 0; i < n; i++) res += a[i]; return res; }
    if (n <= 128) {
        double r[8];
        for (int j = 0; j < 8; j++) r[j] = a[j];
        int i = 8;
        for (; i < n - (n % 8); i += 8) for (int j = 0; j < 8; j++) r[j] += a[i + j];
        double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; i++) res += a[i];
        return res;
    }
    int n2 = n / 2; n2 -= n2 % 8;
    return pairwise_sum(a, n2) + pairwise_sum(a + n2, n - n2);
}

// failure weight of one clip from p = exp(-s / temp) and the sum of p over the C clips (fp32, as failure_weights returns it)
UHC_CDEV float clip_weight(double p, double psum, double freq, int C) { return (float)(freq * (p / psum) + (1.0 - freq) / (double)C); }

// number of entries with percent != 1 in clip c's history
UHC_CDEV int num_failed(const float *pct, const int *meta, int M, int c) {
    int n = 0;
    for (int k = 0; k < meta[2 * c + 1]; k++) n += pct[(size_t)c * M + ring_slot(meta, M, c, k)] != 1.0f;
    return n;
}
// start of the k-th (0-based, oldest first) entry with percent != 1
UHC_CDEV int failed_start(const float *pct, const int *start, const int *meta, int M, int c, int k) {
    for (int j = 0; j < meta[2 * c + 1]; j++) {
        const int s = ring_slot(meta, M, c, j);
        if (pct[(size_t)c * M + s] != 1.0f && k-- == 0) return start[(size_t)c * M + s];
    }
    return 0;
}
// the precision window [lo, hi) around a failed start idx; hi - lo >= 1 (the reference's randint would raise on an empty window,
// which a start recorded from a longer table could produce)
UHC_CDEV void prec_window(int idx, int L, int t_min, int *lo, int *hi) {
    int span = L - t_min; if (span < 1) span = 1;
    int h = idx + PREC_WINDOW < span ? idx + PREC_WINDOW : span;
    if (h < 1) h = 1;
    int l = idx - PREC_WINDOW - t_min > 0 ? idx - PREC_WINDOW - t_min : 0;
    if (l > h - 1) l = h - 1;
    *lo = l; *hi = h;
}
// start frame from three uniforms in [0, 1): u_coin decides the precision branch, u_pick the failed entry, u_start the frame
UHC_CDEV int draw_start(const float *pct, const int *start, const int *meta, int M, int c, int L, int t_min, float prec_freq,
                        float u_coin, float u_pick, float u_start) {
    int lo = 0, hi = L - t_min; if (hi < 1) hi = 1;
    if (pct && prec_freq > 0.f && u_coin < prec_freq) {
        const int nf = num_failed(pct, meta, M, c);
        if (nf > 0) {
            int k = (int)(u_pick * (float)nf); if (k > nf - 1) k = nf - 1;
            prec_window(failed_start(pct, start, meta, M, c, k), L, t_min, &lo, &hi);
        }
    }
    int st = lo + (int)(u_start * (float)(hi - lo)); if (st > hi - 1) st = hi - 1;
    return st;
}

// the global curriculum's payload (uhc_curriculum_stage / uhc_curriculum_update_gathered): every log entry as three fp32 values
// (clip, percent, start), an entry without an ended episode as (-1, 0, 0).  Each rank writes its own slot of a zeroed [world][T][E][3] array,
// so every element of the all-reduce's sum is one rank's value plus zeros, and x + 0 = x in fp32 in any order (a percent of -0 comes back as
// +0, equal under the == the weights use).  Clip indices and start frames are integers, exact in fp32 up to 2^24.
constexpr int STAGE_EXACT_MAX = 1 << 24;
UHC_CDEV bool stage_exact(long long num_clips, long long longest_clip) { return num_clips <= STAGE_EXACT_MAX && longest_clip <= STAGE_EXACT_MAX; }
UHC_CDEV void stage_entry(int clip, float pct, int start, float *out) {
    const bool ended = clip >= 0;
    out[0] = ended ? (float)clip : -1.f; out[1] = ended ? pct : 0.f; out[2] = ended ? (float)start : 0.f;
}
UHC_CDEV void unpack_entry(const float *in, int *clip, float *pct, int *start) { *clip = (int)in[0]; *pct = in[1]; *start = (int)in[2]; }

#ifndef UHC_EMU
// device state of the curriculum (owned by the engine, step_kernel.cu) and the launches of curriculum.cu
struct Dev {
    float *pct; int *start, *meta;      // [C][M], [C][M], [C][2]
    int M, C, t_max;
    double temp, freq;
    float *cdf; const int *clip_adr;    // the sampler's CDF (rewritten in place), the clip table's first frames [C + 1]
    double *p;                          // scratch [C]
    int *cnt, *rank, *ncl;              // scratch of an update: [chunks][C], [N], [C]
};
constexpr int UPD_CHUNK = 1024;         // log entries per block of the bucketing
// bucket the N-entry log (clip_log < 0: no episode ended) into the rings, then the weights and the CDF
cudaError_t launch_update(const Dev &d, const int *clip_log, const float *pct_log, const int *start_log, int N, cudaStream_t st);
// the weights and the CDF from the rings as they are
cudaError_t launch_weights(const Dev &d, cudaStream_t st);
// n log entries -> out [n][3] (stage_entry); the summed payload [n][3] -> the three logs of launch_update (unpack_entry)
cudaError_t launch_stage(const int *clip_log, const float *pct_log, const int *start_log, int n, float *out, cudaStream_t st);
cudaError_t launch_unpack(const float *in, int n, int *clip_log, float *pct_log, int *start_log, cudaStream_t st);
#endif

#ifdef UHC_EMU
// the exact law of draw_start's start frame for clip c (pmf[0 .. L - 1]), with continuous uniforms
static inline void start_law(const float *pct, const int *start, const int *meta, int M, int c, int L, int t_min, double prec_freq, double *pmf) {
    for (int s = 0; s < L; s++) pmf[s] = 0.0;
    const int nf = pct ? num_failed(pct, meta, M, c) : 0;
    const double q = nf > 0 ? prec_freq : 0.0;
    int span = L - t_min; if (span < 1) span = 1;
    for (int s = 0; s < span; s++) pmf[s] += (1.0 - q) / span;
    for (int k = 0; k < nf && q > 0; k++) {
        int lo, hi; prec_window(failed_start(pct, start, meta, M, c, k), L, t_min, &lo, &hi);
        for (int s = lo; s < hi; s++) pmf[s] += q / nf / (hi - lo);
    }
}
#endif

}  // namespace cur
}  // namespace uhc
