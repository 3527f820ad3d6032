// rollout.cu -- the sampling loop behind the C ABI (include/uhc_rollout.h): uhc_policy_forward and uhc_rollout.
//
// Replaces the reference's per-process Python loop  Agent.sample_worker  (uhc/agents/agent_copycat.py:496-571:
//   state -> running_state -> policy_net.select_action -> env.step -> custom_reward -> memory.push(state, action, mask, reward, exp))
// by T lock-step control steps of all E device-resident environments.  One control step is
//   k_zfilter_partial, _merge, _count, k_zfilter_apply_bf16   obs -> normalised state (buffer row, fp32) + bf16 K-padded copy      (a12)
//   4 x k_linear_tc                                           policy MLP on tensor cores (wgmma / TMA, mlp_wgmma.cu)                (a13)
//   k_gauss_sample_dev                                        action + log-prob into the buffer row                                  (a13)
//   k_env_step                                                15 physics substeps + obs + reward + termination + in-kernel re-seeding (a1-a10)
//   k_rollout_post                                            mask / fail / exp rows, device step counter += 1                        (a11)
// and the whole T-step sequence is captured ONCE per (T, buffers, weights) into a CUDA graph (graph_cache.h) and replayed: no host code
// and no torch glue between the kernels.  Everything that varies between replays lives in device memory (the RNG step counter, the ZFilter
// statistics, the env state), so a replay needs no new kernel parameters.
//
// The policy forward (scratch, validation, the walk over nets and layers) is written once here and also serves the evaluation and the
// tracker (eval_glue.h), for one policy over all rows or for several side by side.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../include/uhc_nn.h"
#include "../../include/uhc_rollout.h"
#include "errors.h"
#include "eval_glue.h"
#include "graph_cache.h"
#include "group_core.h"

namespace {

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}
__device__ __forceinline__ float gauss_from(uint64_t seed, uint64_t idx) {   // identical to nn_kernels.cu (same stream of normals as uhc_gaussian_sample)
    const uint64_t h = splitmix64(seed ^ splitmix64(idx));
    const float u1 = ((uint32_t)(h >> 40) + 1.0f) * 0x1.fffffcp-25f, u2 = (uint32_t)(h & 0xFFFFFF) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
// ZFilter apply fused with the bf16 K-padded copy the first GEMM reads: y = clip((x - mean) / (std + 1e-8)) (zfilter.py:59-73);
// arithmetic identical to k_zfilter_apply + k_f32_to_bf16_padded.  Element i = (row r, column j) of the [M][Kp] copy, under the statistics
// `stats` of count n
__device__ __forceinline__ void zfilter_apply_bf16_elem(const float *__restrict__ X, float *__restrict__ Y, unsigned short *__restrict__ Yb, size_t i, size_t r, int j,
                                                        int D, const double *__restrict__ stats, double n, float clip) {
    float y = 0.f;
    if (j < D) {
        const double mean = stats[1 + j], var = n > 1.0 ? stats[1 + D + j] / (n - 1.0) : mean * mean;
        y = (float)(((double)X[r * D + j] - mean) / (sqrt(var) + 1e-8));
        if (clip > 0.f) y = fminf(fmaxf(y, -clip), clip);
        if (Y) Y[r * D + j] = y;
    }
    // round-to-nearest-even bf16 (what __float2bfloat16_rn does)
    unsigned u = __float_as_uint(y);
    unsigned short b = (y != y) ? 0x7FFF : (unsigned short)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
    Yb[i] = b;
}
__global__ void k_zfilter_apply_bf16(const float *__restrict__ X, float *__restrict__ Y, unsigned short *__restrict__ Yb, int M, int D, int Kp,
                                     const double *__restrict__ stats, float clip) {
    const double n = stats[0];
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)M * Kp; i += (size_t)gridDim.x * blockDim.x)
        zfilter_apply_bf16_elem(X, Y, Yb, i, i / Kp, (int)(i % Kp), D, stats, n, clip);
}
// the same with one ZFilter per group of rows (the grouped evaluation: several checkpoints side by side): rows [row0[g], row0[g + 1])
// are normalised by stats[g]
struct ZGroups { const double *stats[uhc::grp::MAX_GROUPS]; int row0[uhc::grp::MAX_GROUPS + 1]; int G; };
__global__ void k_zfilter_apply_bf16_grouped(const float *__restrict__ X, float *__restrict__ Y, unsigned short *__restrict__ Yb, int M, int D, int Kp,
                                             const __grid_constant__ ZGroups zg, float clip) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)M * Kp; i += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % Kp); const size_t r = i / Kp;
        int lo = 0, hi = zg.G - 1;                 // the last group starting at or before row r
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if ((size_t)zg.row0[mid] <= r) lo = mid; else hi = mid - 1; }
        const double *stats = zg.stats[lo];
        zfilter_apply_bf16_elem(X, Y, Yb, i, r, j, D, stats, stats[0], clip);
    }
}
// Bernoulli(1 - noise_rate) per env and step: mean_action flag and the `exp` row (agent_copycat.py:530,551)
__global__ void k_mean_action(unsigned char *__restrict__ mean_action, float *__restrict__ exps_row, int E, float p_mean, uint64_t seed,
                              const unsigned long long *__restrict__ step_ptr) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const uint64_t h = splitmix64((seed * 0x9E3779B97F4A7C15ull) ^ splitmix64(*step_ptr * (uint64_t)E + e + 0x5bd1e995ull));
    const float u = (uint32_t)(h >> 40) * (1.0f / 16777216.0f);
    const unsigned char m = u < p_mean;
    mean_action[e] = m; exps_row[e] = 1.0f - (float)m;
}
// same arithmetic as k_gauss_sample (nn_kernels.cu) with the step counter read from device memory
__global__ void k_gauss_sample_dev(const float *__restrict__ mean, const float *__restrict__ log_std, const uint8_t *__restrict__ mean_action,
                                   float *__restrict__ action, float *__restrict__ logp, int M, int A, uint64_t seed, const unsigned long long *__restrict__ step_ptr) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    const uint64_t step = *step_ptr;
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
// mask = 0 on fail or clip end (agent_copycat.py:550), fail row, exps = 1 when every action is sampled; advances the step counter
__global__ void k_rollout_post(const int *__restrict__ fail, const int *__restrict__ end, float *__restrict__ mask_row, int *__restrict__ fail_row,
                               float *__restrict__ exps_row_or_null, int E, unsigned long long *__restrict__ step_ptr, const int *__restrict__ ep_log,
                               int *__restrict__ ep_clip_row, float *__restrict__ ep_pct_row, int *__restrict__ ep_start_row) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) {
        const int f = fail[e], d = f | end[e];
        mask_row[e] = d ? 0.f : 1.f;
        if (fail_row) fail_row[e] = f;
        if (exps_row_or_null) exps_row_or_null[e] = 1.f;
        if (ep_clip_row) { ep_clip_row[e] = ep_log[2 * e]; ep_pct_row[e] = __int_as_float(ep_log[2 * e + 1]); }
        if (ep_start_row) ep_start_row[e] = ep_log[2 * E + e];
    }
    if (e == 0) *step_ptr += 1ull;   // ordered after every reader of this step's counter by the stream / graph dependencies
}

using uhc::GraphCache;
using uhc::evalx::Policy;

int num_nets(const Policy *pol) { return pol->nprim > 0 ? pol->nprim + 1 : 1; }
int pad64(int n) { return (n + 63) / 64 * 64; }

// every argument of uhc_rollout that reaches a kernel; zeroed, then filled: its bytes are the graph's key
struct GraphKey {
    int T, row0, update_filter; float noise_rate, zclip; unsigned long long seed; Policy pol; UhcRolloutBuf buf; const float *log_std; double *zstats;
    unsigned long long cur_gen;   // the sampler's curriculum view (uhc_curriculum_enable) is captured by value: a new one needs a new graph
};
// the buffers of one policy forward over E rows.  Graphs hold these pointers as kernel parameters, so gen moves whenever one of them is
// reallocated.  Zero filled once: the GEMMs write the first N columns of a K-padded activation only, and the grouped forward leaves the
// rows past its groups alone
struct PolicyScratch {
    struct Net { void *acts[9] = {nullptr}; int ld[9] = {0}; };
    Net ns[UHC_MCP_MAX_PRIM + 1];            // bf16 activations per net of the policy; ns[0].acts[0] (the normalised observation) feeds every net
    float *d_mean = nullptr, *d_log_std0 = nullptr; int mean_cap = 0;   // d_log_std0: zeros, the grouped forward's log_std (its mask is all ones, so
                                                                         // k_gauss_sample_dev writes mean + 1 * 0, what any finite log_std gives)
    float *d_xall = nullptr, *d_comp = nullptr; size_t xall_cap = 0;    // PolicyMCP: primitive outputs [P][E][A], composer outputs [E][P]
    unsigned long long gen = 0;
};
struct RolloutCtx {
    UhcEngine *eng = nullptr; int E = 0, device = 0;
    unsigned long long *d_step = nullptr;
    // two instances that never share an allocation: the rollout's, the single-policy evaluation's and the tracker's graphs hold `own`, the
    // grouped evaluation's graphs hold `grouped`, and either may be resized while graphs over the other stay cached
    PolicyScratch own, grouped;
    double *d_zws = nullptr; int zws_d = 0;
    unsigned char *d_mean_action = nullptr; float *d_cinfo = nullptr, *d_pct = nullptr; int *d_fail = nullptr, *d_end = nullptr;
    GraphCache graphs{64};
    int launches_per_step = 0;
    std::vector<cudaEvent_t> ev0, ev1;    // optional: events around the env-step kernel of buffer row r (bench roofline: the dominant kernel's live duration)
};
std::vector<RolloutCtx *> g_ctx;

RolloutCtx *ctx_of(UhcEngine *e) {
    for (RolloutCtx *c : g_ctx) if (c->eng == e) return c;
    RolloutCtx *c = new RolloutCtx(); c->eng = e; c->E = uhc_num_envs(e);
    g_ctx.push_back(c);
    return c;
}

int check_policy(const Policy *pol) {
    const int P = pol->nprim;
    if (P < 0 || P > UHC_MCP_MAX_PRIM) { uhc_err() = "UhcMcp: 1..8 primitives"; return -2; }
    const UhcMlp *m0 = &pol->nets[0];
    for (int j = 0; j < num_nets(pol); j++) {
        const UhcMlp *m = &pol->nets[j];
        if (m->nlayers < 1 || m->nlayers > 8) { uhc_err() = "UhcMlp: 1..8 layers"; return -2; }
        if (m->dims[0] != m0->dims[0]) { uhc_err() = "UhcMcp: every net reads the same observation"; return -2; }
        if (j < P && m->dims[m->nlayers] != m0->dims[m0->nlayers]) { uhc_err() = "UhcMcp: the primitives must share the action width"; return -2; }
        if (P > 0 && j == P && m->dims[m->nlayers] != P) { uhc_err() = "UhcMcp: the composer's output width must be the number of primitives"; return -2; }
        for (int i = 0; i < m->nlayers; i++) {
            if (m->kp[i] != pad64(m->dims[i])) { uhc_err() = "UhcMlp: kp[i] must be dims[i] rounded up to 64"; return -2; }
            if (!m->W_bf16[i]) { uhc_err() = "UhcMlp: null weights"; return -2; }
        }
    }
    return 0;
}

int realloc_zero(void **p, size_t bytes) {
    if (*p) { cudaFree(*p); *p = nullptr; }
    CK(cudaMalloc(p, bytes)); CK(cudaMemset(*p, 0, bytes));
    return 0;
}
// validates pol (-2, nothing touched) and sizes s for it over E rows
int ensure(PolicyScratch *s, size_t E, const Policy *pol) {
    if (const int rc = check_policy(pol)) return rc;
    const UhcMlp *m0 = &pol->nets[0];
    const size_t P = pol->nprim, A = m0->dims[m0->nlayers];
    for (int j = 0; j < num_nets(pol); j++) {
        const UhcMlp *m = &pol->nets[j];
        for (int i = 0; i < m->nlayers; i++) {
            if ((i == 0 && j > 0) || s->ns[j].ld[i] == m->kp[i]) continue;       // the input is shared
            s->gen++; s->ns[j].ld[i] = 0;
            if (realloc_zero(&s->ns[j].acts[i], E * m->kp[i] * 2)) return -1;
            s->ns[j].ld[i] = m->kp[i];
        }
    }
    if ((size_t)s->mean_cap < A) {
        s->gen++; s->mean_cap = 0;
        if (realloc_zero((void **)&s->d_mean, E * A * 4) || realloc_zero((void **)&s->d_log_std0, A * 4)) return -1;
        s->mean_cap = (int)A;
    }
    if (P > 0 && s->xall_cap < P * E * A) {
        s->gen++; s->xall_cap = 0;
        if (realloc_zero((void **)&s->d_xall, P * E * A * 4) || realloc_zero((void **)&s->d_comp, E * UHC_MCP_MAX_PRIM * 4)) return -1;
        s->xall_cap = P * E * A;
    }
    return 0;
}
void release(PolicyScratch *s) {
    for (auto &nsj : s->ns) for (void *p : nsj.acts) if (p) cudaFree(p);
    for (void *p : {(void *)s->d_mean, (void *)s->d_log_std0, (void *)s->d_xall, (void *)s->d_comp}) if (p) cudaFree(p);
}
// the step counter and the per-env arrays of the context: allocated once, never moved
int ensure_ctx(RolloutCtx *c) {
    const size_t E = c->E;
    if (!c->d_step) { CK(cudaMalloc((void **)&c->d_step, sizeof(unsigned long long))); CK(cudaMemset(c->d_step, 0, sizeof(unsigned long long))); }
    if (!c->d_mean_action) {
        CK(cudaMalloc((void **)&c->d_mean_action, E)); CK(cudaMalloc((void **)&c->d_cinfo, E * 5 * 4)); CK(cudaMalloc((void **)&c->d_pct, E * 4));
        CK(cudaMalloc((void **)&c->d_fail, E * 4)); CK(cudaMalloc((void **)&c->d_end, E * 4));
    }
    return 0;
}
// the context's own scratch for pol.  Its graphs hold those pointers, so a reallocation drops them all; own.gen (the evaluation's and the
// tracker's graphs hold the same pointers) has moved then
int ensure_own(RolloutCtx *c, const Policy *pol) {
    const unsigned long long gen0 = c->own.gen;
    int rc = ensure_ctx(c);
    if (!rc) rc = ensure(&c->own, c->E, pol);
    const int D = pol->nets[0].dims[0];
    if (!rc && c->zws_d < D) {
        c->own.gen++; c->zws_d = 0;
        rc = realloc_zero((void **)&c->d_zws, (size_t)uhc_zfilter_workspace_doubles(D) * sizeof(double));
        if (!rc) c->zws_d = D;
    }
    if (c->own.gen != gen0) c->graphs.clear();
    return rc;
}

// One layer of the walk below: the GEMM in [E][Kp] bf16 -> N columns, into the next bf16 activation (leading dimension ld) or, for a
// net's last layer, into its fp32 output
struct Layer { int net, i; const void *in; void *out_bf16; float *out_f32; int N, Kp, ld, act; };
// the policy's nets layer by layer over the scratch s, then the mixture head: MLP -> d_mean; PolicyMCP: primitives -> d_xall, composer
// (+ softmax) -> d_comp, weighted sum -> d_mean.  gemm(Layer) enqueues one layer.  Returns the number of kernels enqueued (or < 0).
template <class Gemm>
int enqueue_layers(const PolicyScratch &s, const Policy *pol, int E, cudaStream_t st, Gemm &&gemm) {
    const UhcMlp *m0 = &pol->nets[0];
    const int P = pol->nprim, A = m0->dims[m0->nlayers];
    int n = 0;
    for (int j = 0; j < num_nets(pol); j++) {
        const UhcMlp *m = &pol->nets[j];
        const bool composer = P > 0 && j == P;
        float *out = P == 0 ? s.d_mean : (composer ? s.d_comp : s.d_xall + (size_t)j * E * A);
        for (int i = 0; i < m->nlayers; i++) {
            const bool last = i == m->nlayers - 1;
            // the composer is a plain MLP (mlp.py:24-27): its last affine layer is followed by the activation too, then the softmax (policy_mcp.py:26)
            const Layer l{j, i, i == 0 ? s.ns[0].acts[0] : s.ns[j].acts[i], last ? nullptr : s.ns[j].acts[i + 1], last ? out : nullptr, m->dims[i + 1], m->kp[i],
                          last ? 0 : s.ns[j].ld[i + 1], (last && !composer) ? UHC_ACT_NONE : m->act};
            if (gemm(l)) return -1;
            n++;
        }
    }
    // the mixture head is row-wise: run over every row (a row no policy covers holds zeros or earlier values and is never read)
    if (P > 0) { if (uhc_mcp_combine(s.d_xall, s.d_comp, nullptr, s.d_mean, E, A, P, st)) return uhc_err_prefix("mixture head"); n++; }
    return n;
}

// obs -> (state row, bf16 copy) -> policy -> mean (the context's own scratch).  Returns the number of kernels enqueued (or < 0).
int enqueue_policy(RolloutCtx *c, const float *obs, const Policy *pol, double *zstats, float zclip, int update_filter, float *state_out, cudaStream_t st) {
    const UhcMlp *m0 = &pol->nets[0];
    const int E = c->E, D = m0->dims[0];
    int n = 0;
    if (update_filter) { if (uhc_zfilter_ws(obs, nullptr, E, D, zstats, zclip, 1, c->d_zws, st)) return uhc_err_prefix("zfilter update"); n += 3; }
    k_zfilter_apply_bf16<<<1056, 256, 0, st>>>(obs, state_out, (unsigned short *)c->own.ns[0].acts[0], E, D, m0->kp[0], zstats, zclip);
    CK(cudaGetLastError()); n++;
    const int nl = enqueue_layers(c->own, pol, E, st, [&](const Layer &l) {
        const UhcMlp *m = &pol->nets[l.net];
        return uhc_linear_forward_tc(l.in, m->W_bf16[l.i], m->bias[l.i], l.out_bf16, l.out_f32, E, l.N, l.Kp, l.ld, l.act, st) ? uhc_err_prefix("policy GEMM") : 0;
    });
    return nl < 0 ? nl : n + nl;
}

int enqueue_step(RolloutCtx *c, int row, const Policy *pol, const float *log_std, double *zstats, float zclip, int update_filter, unsigned long long seed,
                 float noise_rate, const UhcRolloutBuf *b, cudaStream_t st) {
    const UhcMlp *m = &pol->nets[0];
    const size_t E = c->E; const int D = m->dims[0], A = m->dims[m->nlayers];
    float *state_row = b->states + (size_t)row * E * D, *act_row = b->actions + (size_t)row * E * A;
    float *rew_row = b->rewards + (size_t)row * E, *mask_row = b->masks + (size_t)row * E, *exps_row = b->exps + (size_t)row * E;
    float *logp_row = b->logp ? b->logp + (size_t)row * E : nullptr; int *fail_row = b->fails ? b->fails + (size_t)row * E : nullptr;
    int n = enqueue_policy(c, b->obs_cur, pol, zstats, zclip, update_filter, state_row, st);
    if (n < 0) return n;
    const bool mixed = noise_rate < 1.0f;
    if (mixed) { k_mean_action<<<(c->E + 255) / 256, 256, 0, st>>>(c->d_mean_action, exps_row, c->E, 1.0f - noise_rate, seed, c->d_step); CK(cudaGetLastError()); n++; }
    k_gauss_sample_dev<<<(c->E + 7) / 8, 256, 0, st>>>(c->own.d_mean, log_std, mixed ? c->d_mean_action : nullptr, act_row, logp_row, c->E, A, seed, c->d_step);
    CK(cudaGetLastError()); n++;
    const bool timed = row < (int)c->ev0.size();
    // inside stream capture the record must be an EXTERNAL event-record node, or the event is owned by the graph and cannot be read from the host
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (timed) CK(cudaStreamIsCapturing(st, &cap));
    const unsigned evflag = cap == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault;
    if (timed) CK(cudaEventRecordWithFlags(c->ev0[row], st, evflag));
    if (uhc_env_step(c->eng, act_row, b->obs_cur, rew_row, c->d_cinfo, c->d_fail, c->d_end, c->d_pct, nullptr, st)) return uhc_err_prefix("env step");
    if (timed) CK(cudaEventRecordWithFlags(c->ev1[row], st, evflag));
    n++;
    const bool eplog = b->ep_clip && b->ep_pct;
    k_rollout_post<<<(c->E + 255) / 256, 256, 0, st>>>(c->d_fail, c->d_end, mask_row, fail_row, mixed ? nullptr : exps_row, c->E, c->d_step, uhc_episode_log_dev(c->eng),
                                                       eplog ? b->ep_clip + (size_t)row * E : nullptr, eplog ? b->ep_pct + (size_t)row * E : nullptr,
                                                       eplog && b->ep_start ? b->ep_start + (size_t)row * E : nullptr);
    CK(cudaGetLastError()); n++;
    return n;
}

}  // namespace

extern "C" {

int uhc_rollout_set_step(UhcEngine *e, unsigned long long step) {
    if (!e) { uhc_err() = "uhc_rollout_set_step: null engine"; return -2; }
    RolloutCtx *c = ctx_of(e);
    if (!c->d_step) { CK(cudaMalloc((void **)&c->d_step, sizeof(unsigned long long))); }
    CK(cudaMemcpy(c->d_step, &step, sizeof step, cudaMemcpyHostToDevice));
    return 0;
}
int uhc_rollout_get_step(UhcEngine *e, unsigned long long *step) {
    if (!e || !step) { uhc_err() = "uhc_rollout_get_step: bad argument"; return -2; }
    RolloutCtx *c = ctx_of(e);
    *step = 0;
    if (c->d_step) { CK(cudaDeviceSynchronize()); CK(cudaMemcpy(step, c->d_step, sizeof *step, cudaMemcpyDeviceToHost)); }
    return 0;
}

static int make_policy(Policy *pol, const UhcMlp *mlp, const UhcMcp *mcp, UhcEngine *e, const char *who) {
    memset(pol, 0, sizeof *pol);
    if (mcp) {
        if (mcp->nprim < 1 || mcp->nprim > UHC_MCP_MAX_PRIM) { uhc_err() = std::string(who) + ": 1..8 primitives"; return -2; }
        pol->nprim = mcp->nprim;
        for (int k = 0; k < mcp->nprim; k++) pol->nets[k] = mcp->prim[k];
        pol->nets[mcp->nprim] = mcp->composer;
    } else pol->nets[0] = *mlp;
    const UhcMlp *m = &pol->nets[0];
    if (m->nlayers >= 1 && m->nlayers <= 8 && (m->dims[m->nlayers] != uhc_engine_act_dim(e) || m->dims[0] != uhc_engine_obs_dim(e))) {
        uhc_err() = std::string(who) + ": the policy's input / output widths are not the engine's obs / action dims"; return -2;
    }
    return 0;
}
static int policy_forward_impl(UhcEngine *e, const float *obs_dev, const Policy *pol, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                               unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                               void *stream) {
    RolloutCtx *c = ctx_of(e);
    int rc = ensure_own(c, pol);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (enqueue_policy(c, obs_dev, pol, zfilter_stats, zclip, update_filter, state_out_or_null, st) < 0) return -1;
    const UhcMlp *m = &pol->nets[0];
    k_gauss_sample_dev<<<(c->E + 7) / 8, 256, 0, st>>>(c->own.d_mean, log_std, mean_action_or_null, action_out, logp_out_or_null, c->E, m->dims[m->nlayers], seed, c->d_step);
    CK(cudaGetLastError());
    return 0;
}
static int rollout_impl(UhcEngine *e, int T, int row0, const Policy *pol, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                        unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream) {
    RolloutCtx *c = ctx_of(e);
    int rc = ensure_own(c, pol);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (!use_graph) {
        for (int k = 0; k < T; k++) { const int n = enqueue_step(c, row0 + k, pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, st); if (n < 0) return -1; c->launches_per_step = n; }
        return 0;
    }
    GraphKey k; memset(&k, 0, sizeof k);
    k.T = T; k.row0 = row0; k.update_filter = update_filter; k.noise_rate = noise_rate; k.zclip = zclip; k.seed = seed; k.pol = *pol; k.buf = *buf;
    k.log_std = log_std; k.zstats = zfilter_stats; k.cur_gen = uhc::evalx::curriculum_gen(e);
    std::string key; GraphCache::append(&key, &k);
    cudaGraphExec_t exec = c->graphs.find(key);
    if (!exec) {
        int n = 0;
        rc = GraphCache::capture([&](cudaStream_t cs) {
            for (int i = 0; i < T && n >= 0; i++) n = enqueue_step(c, row0 + i, pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, cs);
            return n < 0 ? -1 : 0;
        }, &exec);
        if (rc) return rc;
        c->launches_per_step = n;
        c->graphs.insert(std::move(key), GraphCache::Gens{}, exec);   // nothing goes stale: the scratch drops them all, the rest is in the key
    }
    CK(cudaGraphLaunch(exec, st));
    return 0;
}

int uhc_policy_forward(UhcEngine *e, const float *obs_dev, const UhcMlp *mlp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                       unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                       void *stream) {
    if (!e || !obs_dev || !mlp || !log_std || !zfilter_stats || !action_out) { uhc_err() = "uhc_policy_forward: bad argument"; return -2; }
    Policy pol; if (make_policy(&pol, mlp, nullptr, e, "uhc_policy_forward")) return -2;
    return policy_forward_impl(e, obs_dev, &pol, log_std, zfilter_stats, zclip, update_filter, seed, mean_action_or_null, state_out_or_null, action_out, logp_out_or_null, stream);
}
int uhc_policy_forward_mcp(UhcEngine *e, const float *obs_dev, const UhcMcp *mcp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                           unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                           void *stream) {
    if (!e || !obs_dev || !mcp || !log_std || !zfilter_stats || !action_out) { uhc_err() = "uhc_policy_forward_mcp: bad argument"; return -2; }
    Policy pol; if (make_policy(&pol, nullptr, mcp, e, "uhc_policy_forward_mcp")) return -2;
    return policy_forward_impl(e, obs_dev, &pol, log_std, zfilter_stats, zclip, update_filter, seed, mean_action_or_null, state_out_or_null, action_out, logp_out_or_null, stream);
}

int uhc_rollout(UhcEngine *e, int T, int row0, const UhcMlp *mlp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream) {
    if (!e || !mlp || !log_std || !zfilter_stats || !buf || T <= 0 || row0 < 0 || row0 + T > buf->T_cap) { uhc_err() = "uhc_rollout: bad argument"; return -2; }
    if (!buf->states || !buf->actions || !buf->rewards || !buf->masks || !buf->exps || !buf->obs_cur) { uhc_err() = "uhc_rollout: missing buffer"; return -2; }
    Policy pol; if (make_policy(&pol, mlp, nullptr, e, "uhc_rollout")) return -2;
    return rollout_impl(e, T, row0, &pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, use_graph, stream);
}
int uhc_rollout_mcp(UhcEngine *e, int T, int row0, const UhcMcp *mcp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                    unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream) {
    if (!e || !mcp || !log_std || !zfilter_stats || !buf || T <= 0 || row0 < 0 || row0 + T > buf->T_cap) { uhc_err() = "uhc_rollout_mcp: bad argument"; return -2; }
    if (!buf->states || !buf->actions || !buf->rewards || !buf->masks || !buf->exps || !buf->obs_cur) { uhc_err() = "uhc_rollout_mcp: missing buffer"; return -2; }
    Policy pol; if (make_policy(&pol, nullptr, mcp, e, "uhc_rollout_mcp")) return -2;
    return rollout_impl(e, T, row0, &pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, use_graph, stream);
}

// events around the env-step kernel of rows 0 .. nrows-1 (recorded on the launching stream, also inside graph replays); 0 disables.
// Changing it drops the cached graphs.
int uhc_rollout_time_env_step(UhcEngine *e, int nrows) {
    if (!e || nrows < 0) { uhc_err() = "uhc_rollout_time_env_step: bad argument"; return -2; }
    RolloutCtx *c = ctx_of(e);
    CK(cudaDeviceSynchronize());
    c->graphs.clear();
    for (cudaEvent_t ev : c->ev0) cudaEventDestroy(ev);
    for (cudaEvent_t ev : c->ev1) cudaEventDestroy(ev);
    c->ev0.assign(nrows, nullptr); c->ev1.assign(nrows, nullptr);
    for (int i = 0; i < nrows; i++) { CK(cudaEventCreate(&c->ev0[i])); CK(cudaEventCreate(&c->ev1[i])); }
    return 0;
}
int uhc_rollout_env_step_ms(UhcEngine *e, int row, float *ms) {
    if (!e || !ms) { uhc_err() = "uhc_rollout_env_step_ms: bad argument"; return -2; }
    RolloutCtx *c = ctx_of(e);
    if (row < 0 || row >= (int)c->ev0.size()) { uhc_err() = "uhc_rollout_env_step_ms: row not timed"; return -2; }
    CK(cudaEventSynchronize(c->ev1[row]));
    CK(cudaEventElapsedTime(ms, c->ev0[row], c->ev1[row]));
    return 0;
}

int uhc_rollout_launches_per_step(UhcEngine *e) { return e ? ctx_of(e)->launches_per_step : -1; }

}  // extern "C"

void uhc::evalx::drop_rollout_graphs(UhcEngine *e) {
    for (RolloutCtx *c : g_ctx) if (c->eng == e) c->graphs.clear();
}

extern "C" {

void uhc_rollout_release(UhcEngine *e) {   // called by the binding before uhc_engine_destroy
    for (size_t i = 0; i < g_ctx.size(); i++) if (g_ctx[i]->eng == e) {
        RolloutCtx *c = g_ctx[i];
        c->graphs.clear();
        for (cudaEvent_t ev : c->ev0) cudaEventDestroy(ev);
        for (cudaEvent_t ev : c->ev1) cudaEventDestroy(ev);
        release(&c->own); release(&c->grouped);
        for (void *p : {(void *)c->d_zws, (void *)c->d_step, (void *)c->d_mean_action, (void *)c->d_cinfo, (void *)c->d_pct, (void *)c->d_fail, (void *)c->d_end}) if (p) cudaFree(p);
        delete c; g_ctx.erase(g_ctx.begin() + i); return;
    }
}

}  // extern "C"

// ---- the policy forward of the device evaluation and the tracker (eval_glue.h): the kernels of uhc_policy_forward(_mcp), enqueued from
// eval.cu's and track.cu's graphs
namespace uhc {
namespace evalx {

int policy_prepare(UhcEngine *e, const UhcMlp *mlp, const UhcMcp *mcp, Policy *pol, unsigned long long *gen) {
    if (make_policy(pol, mlp, mcp, e, mcp ? "uhc_eval_run_mcp" : "uhc_eval_run")) return -2;
    RolloutCtx *c = ctx_of(e);
    const int rc = ensure_own(c, pol);
    *gen = c->own.gen;
    return rc;
}

int policy_enqueue(UhcEngine *e, const Policy &pol, const float *obs, const float *log_std, double *zstats, float zclip, const unsigned char *mean_action,
                   float *action, cudaStream_t st) {
    RolloutCtx *c = ctx_of(e);
    if (enqueue_policy(c, obs, &pol, zstats, zclip, 0, nullptr, st) < 0) return -1;
    const UhcMlp *m = &pol.nets[0];
    k_gauss_sample_dev<<<(c->E + 7) / 8, 256, 0, st>>>(c->own.d_mean, log_std, mean_action, action, nullptr, c->E, m->dims[m->nlayers], 0, c->d_step);
    CK(cudaGetLastError());
    return 0;
}

// ---- the grouped policy forward of uhc_eval_run_groups: G policies of one architecture over consecutive row ranges of the context's
// second scratch
namespace {
// every group's policy must have group 0's architecture: primitive count, and per net the layer count, activation, widths and K padding
bool same_arch(const Policy *a, const Policy *b) {
    if (a->nprim != b->nprim) return false;
    for (int j = 0; j < num_nets(a); j++) {
        const UhcMlp &x = a->nets[j], &y = b->nets[j];
        if (x.nlayers != y.nlayers || x.act != y.act) return false;
        for (int i = 0; i <= x.nlayers; i++) if (x.dims[i] != y.dims[i]) return false;
        for (int i = 0; i < x.nlayers; i++) if (x.kp[i] != y.kp[i]) return false;
    }
    return true;
}
}  // namespace

int groups_prepare(UhcEngine *e, int G, const UhcMlp *mlps, const UhcMcp *mcps, std::vector<Policy> *pols, unsigned long long *gen) {
    const char *who = mcps ? "uhc_eval_run_groups_mcp" : "uhc_eval_run_groups";
    pols->resize(G);
    for (int g = 0; g < G; g++) {
        Policy *p = &(*pols)[g];
        if (make_policy(p, mlps ? mlps + g : nullptr, mcps ? mcps + g : nullptr, e, who)) return -2;
        if (check_policy(p)) { uhc_err_prefix(who); return -2; }
        if (g > 0 && !same_arch(&(*pols)[0], p)) { uhc_err() = std::string(who) + ": every group's policy must have the same layer widths, K padding, activation and primitive count"; return -2; }
    }
    RolloutCtx *c = ctx_of(e);
    int rc = ensure_ctx(c);
    if (!rc) rc = ensure(&c->grouped, c->E, &(*pols)[0]);
    *gen = c->grouped.gen;
    return rc;
}

int groups_enqueue(UhcEngine *e, const std::vector<Policy> &pols, const int *row0, const double *const *zstats, float zclip, const float *obs,
                   const unsigned char *mean_action, float *action, cudaStream_t st) {
    RolloutCtx *c = ctx_of(e);
    const PolicyScratch &s = c->grouped;
    const UhcMlp *m0 = &pols[0].nets[0];
    const int G = (int)pols.size(), ntot = row0[G];
    ZGroups zg;
    memset(&zg, 0, sizeof zg);
    zg.G = G;
    int rows[uhc::grp::MAX_GROUPS];
    for (int g = 0; g <= G; g++) zg.row0[g] = row0[g];
    for (int g = 0; g < G; g++) { zg.stats[g] = zstats[g]; rows[g] = row0[g + 1] - row0[g]; }
    k_zfilter_apply_bf16_grouped<<<1056, 256, 0, st>>>(obs, nullptr, (unsigned short *)s.ns[0].acts[0], ntot, m0->dims[0], m0->kp[0], zg, zclip);
    CK(cudaGetLastError());
    const int nl = enqueue_layers(s, &pols[0], c->E, st, [&](const Layer &l) {
        const void *W[uhc::grp::MAX_GROUPS]; const float *b[uhc::grp::MAX_GROUPS];
        for (int g = 0; g < G; g++) { W[g] = pols[g].nets[l.net].W_bf16[l.i]; b[g] = pols[g].nets[l.net].bias[l.i]; }
        return uhc_linear_forward_tc_grouped(G, row0, rows, l.in, W, b, l.out_bf16, l.out_f32, c->E, l.N, l.Kp, l.ld, l.act, st) ? uhc_err_prefix("grouped policy GEMM") : 0;
    });
    if (nl < 0) return -1;
    k_gauss_sample_dev<<<(ntot + 7) / 8, 256, 0, st>>>(s.d_mean, s.d_log_std0, mean_action, action, nullptr, ntot, m0->dims[m0->nlayers], 0, c->d_step);
    CK(cudaGetLastError());
    return 0;
}

}  // namespace evalx
}  // namespace uhc
