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
// and the whole T-step sequence is captured ONCE per (T, buffers, weights) into a CUDA graph and replayed: no host code and no torch
// glue between the kernels.  Everything that varies between replays lives in device memory (the RNG step counter, the ZFilter
// statistics, the env state), so a replay needs no new kernel parameters.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../include/uhc_nn.h"
#include "../../include/uhc_rollout.h"
#include "eval_glue.h"
#include "group_core.h"

static thread_local std::string g_ro_err;
#define CKR(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { g_ro_err = std::string(#x) + ": " + cudaGetErrorString(e_); return -1; } } while (0)
#define CKC(x, msg) do { if ((x) != 0) { g_ro_err = std::string(msg) + ": " + (uhc_nn_last_error()[0] ? uhc_nn_last_error() : uhc_tc_last_error()); return -1; } } while (0)

extern "C" const char *uhc_tc_last_error(void);

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
// arithmetic identical to k_zfilter_apply + k_f32_to_bf16_padded
__global__ void k_zfilter_apply_bf16(const float *__restrict__ X, float *__restrict__ Y, unsigned short *__restrict__ Yb, int M, int D, int Kp,
                                     const double *__restrict__ stats, float clip) {
    const double n = stats[0];
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)M * Kp; i += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % Kp); const size_t r = i / Kp;
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
}
// the same with one ZFilter per group of rows (the grouped evaluation: several checkpoints side by side): rows [row0[g], row0[g + 1])
// are normalised by stats[g], with k_zfilter_apply_bf16's arithmetic
struct ZGroups { const double *stats[uhc::grp::MAX_GROUPS]; int row0[uhc::grp::MAX_GROUPS + 1]; int G; };
__global__ void k_zfilter_apply_bf16_grouped(const float *__restrict__ X, float *__restrict__ Y, unsigned short *__restrict__ Yb, int M, int D, int Kp,
                                             const __grid_constant__ ZGroups zg, float clip) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)M * Kp; i += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % Kp); const size_t r = i / Kp;
        int lo = 0, hi = zg.G - 1;                 // the last group starting at or before row r
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if ((size_t)zg.row0[mid] <= r) lo = mid; else hi = mid - 1; }
        const double *stats = zg.stats[lo];
        const double n = stats[0];
        float y = 0.f;
        if (j < D) {
            const double mean = stats[1 + j], var = n > 1.0 ? stats[1 + D + j] / (n - 1.0) : mean * mean;
            y = (float)(((double)X[r * D + j] - mean) / (sqrt(var) + 1e-8));
            if (clip > 0.f) y = fminf(fmaxf(y, -clip), clip);
            if (Y) Y[r * D + j] = y;
        }
        unsigned u = __float_as_uint(y);
        unsigned short b = (y != y) ? 0x7FFF : (unsigned short)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
        Yb[i] = b;
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

// the policy of a rollout: one MLP (PolicyGaussian, nprim = 0: nets[0]) or a PolicyMCP mixture (nets[0 .. nprim-1] = primitives, nets[nprim] = composer)
struct Policy { int nprim; int pad; UhcMlp nets[UHC_MCP_MAX_PRIM + 1]; };
struct GraphKey {
    int T, row0, update_filter; float noise_rate, zclip; unsigned long long seed; Policy pol; UhcRolloutBuf buf; const float *log_std; double *zstats;
    unsigned long long cur_gen;   // the sampler's curriculum view (uhc_curriculum_enable) is captured by value: a new one needs a new graph
    bool operator==(const GraphKey &o) const { return memcmp(this, &o, sizeof(GraphKey)) == 0; }
};
struct RolloutCtx {
    UhcEngine *eng = nullptr; int E = 0, device = 0;
    unsigned long long *d_step = nullptr;
    struct NetScratch { void *acts[9] = {nullptr}; int ld[9] = {0}; };
    NetScratch ns[UHC_MCP_MAX_PRIM + 1];     // bf16 activations per net of the policy; ns[0].acts[0] (the normalised observation) feeds every net
    float *d_mean = nullptr; int mean_cap = 0;
    float *d_xall = nullptr, *d_comp = nullptr; size_t xall_cap = 0;   // PolicyMCP: primitive outputs [P][E][A], composer outputs [E][P]
    double *d_zws = nullptr; int zws_d = 0;
    unsigned char *d_mean_action = nullptr; float *d_cinfo = nullptr, *d_pct = nullptr; int *d_fail = nullptr, *d_end = nullptr;
    std::vector<std::pair<GraphKey, cudaGraphExec_t>> graphs;
    unsigned long long scratch_gen = 0;   // bumped whenever the scratch above is reallocated (the evaluation's graphs hold its pointers)
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
int pad64(int n) { return (n + 63) / 64 * 64; }

int ensure_scratch(RolloutCtx *c, const Policy *pol) {
    const size_t E = c->E;
    if (!c->d_step) { CKR(cudaMalloc((void **)&c->d_step, sizeof(unsigned long long))); CKR(cudaMemset(c->d_step, 0, sizeof(unsigned long long))); }
    if (!c->d_mean_action) {
        CKR(cudaMalloc((void **)&c->d_mean_action, E)); CKR(cudaMalloc((void **)&c->d_cinfo, E * 5 * 4)); CKR(cudaMalloc((void **)&c->d_pct, E * 4));
        CKR(cudaMalloc((void **)&c->d_fail, E * 4)); CKR(cudaMalloc((void **)&c->d_end, E * 4));
    }
    const int P = pol->nprim, nnets = P > 0 ? P + 1 : 1;
    if (P < 0 || P > UHC_MCP_MAX_PRIM) { g_ro_err = "UhcMcp: 1..8 primitives"; return -2; }
    const UhcMlp *m0 = &pol->nets[0];
    auto drop_graphs = [&]() { for (auto &g : c->graphs) cudaGraphExecDestroy(g.second); c->graphs.clear(); c->scratch_gen++; };
    for (int j = 0; j < nnets; j++) {
        const UhcMlp *m = &pol->nets[j];
        if (m->nlayers < 1 || m->nlayers > 8) { g_ro_err = "UhcMlp: 1..8 layers"; return -2; }
        if (m->dims[0] != m0->dims[0]) { g_ro_err = "UhcMcp: every net reads the same observation"; return -2; }
        if (j < P && m->dims[m->nlayers] != m0->dims[m0->nlayers]) { g_ro_err = "UhcMcp: the primitives must share the action width"; return -2; }
        if (P > 0 && j == P && m->dims[m->nlayers] != P) { g_ro_err = "UhcMcp: the composer's output width must be the number of primitives"; return -2; }
        for (int i = 0; i < m->nlayers; i++) {   // bf16 activations, K padded to 64 and zero filled once (the GEMMs write the first N columns only)
            const int ld = pad64(m->dims[i]);
            if (m->kp[i] != ld) { g_ro_err = "UhcMlp: kp[i] must be dims[i] rounded up to 64"; return -2; }
            if (i == 0 && j > 0) continue;       // the input is shared
            if (c->ns[j].ld[i] != ld) {
                if (c->ns[j].acts[i]) cudaFree(c->ns[j].acts[i]);
                CKR(cudaMalloc(&c->ns[j].acts[i], E * ld * 2)); CKR(cudaMemset(c->ns[j].acts[i], 0, E * ld * 2));
                c->ns[j].ld[i] = ld;
                drop_graphs();
            }
        }
    }
    if (c->zws_d < m0->dims[0]) {
        if (c->d_zws) cudaFree(c->d_zws);
        CKR(cudaMalloc((void **)&c->d_zws, (size_t)uhc_zfilter_workspace_doubles(m0->dims[0]) * sizeof(double))); c->zws_d = m0->dims[0];
        drop_graphs();
    }
    const int A = m0->dims[m0->nlayers];
    if (c->mean_cap < A) { if (c->d_mean) cudaFree(c->d_mean); CKR(cudaMalloc((void **)&c->d_mean, E * A * 4)); c->mean_cap = A; drop_graphs(); }
    if (P > 0 && c->xall_cap < (size_t)P * E * A) {
        if (c->d_xall) cudaFree(c->d_xall);
        if (c->d_comp) cudaFree(c->d_comp);
        CKR(cudaMalloc((void **)&c->d_xall, (size_t)P * E * A * 4)); CKR(cudaMalloc((void **)&c->d_comp, E * UHC_MCP_MAX_PRIM * 4)); c->xall_cap = (size_t)P * E * A;
        drop_graphs();
    }
    return 0;
}

// obs -> (state row, bf16 copy) -> MLP (or the PolicyMCP mixture: primitives, composer + softmax, weighted sum) -> mean (ctx scratch).
// Returns the number of kernels enqueued (or < 0).
int enqueue_policy(RolloutCtx *c, const float *obs, const Policy *pol, double *zstats, float zclip, int update_filter, float *state_out, cudaStream_t st) {
    const UhcMlp *m0 = &pol->nets[0];
    const int E = c->E, D = m0->dims[0], P = pol->nprim, A = m0->dims[m0->nlayers];
    int n = 0;
    if (update_filter) { CKC(uhc_zfilter_ws(obs, nullptr, E, D, zstats, zclip, 1, c->d_zws, st), "zfilter update"); n += 3; }
    k_zfilter_apply_bf16<<<1056, 256, 0, st>>>(obs, state_out, (unsigned short *)c->ns[0].acts[0], E, D, m0->kp[0], zstats, zclip);
    CKR(cudaGetLastError()); n++;
    for (int j = 0; j < (P > 0 ? P + 1 : 1); j++) {
        const UhcMlp *m = &pol->nets[j];
        const bool composer = P > 0 && j == P;
        float *out = P == 0 ? c->d_mean : (composer ? c->d_comp : c->d_xall + (size_t)j * E * A);
        for (int i = 0; i < m->nlayers; i++) {
            const bool last = i == m->nlayers - 1;
            const void *in = i == 0 ? c->ns[0].acts[0] : c->ns[j].acts[i];
            // the composer is a plain MLP (mlp.py:24-27): its last affine layer is followed by the activation too, then the softmax (policy_mcp.py:26)
            CKC(uhc_linear_forward_tc(in, m->W_bf16[i], m->bias[i], last ? nullptr : c->ns[j].acts[i + 1], last ? out : nullptr, E, m->dims[i + 1], m->kp[i],
                                      last ? 0 : c->ns[j].ld[i + 1], (last && !composer) ? UHC_ACT_NONE : m->act, st), "policy GEMM");
            n++;
        }
    }
    if (P > 0) { CKC(uhc_mcp_combine(c->d_xall, c->d_comp, nullptr, c->d_mean, E, A, P, st), "mixture head"); n++; }
    return n;
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
    if (mixed) { k_mean_action<<<(c->E + 255) / 256, 256, 0, st>>>(c->d_mean_action, exps_row, c->E, 1.0f - noise_rate, seed, c->d_step); CKR(cudaGetLastError()); n++; }
    k_gauss_sample_dev<<<(c->E + 7) / 8, 256, 0, st>>>(c->d_mean, log_std, mixed ? c->d_mean_action : nullptr, act_row, logp_row, c->E, A, seed, c->d_step);
    CKR(cudaGetLastError()); n++;
    const bool timed = row < (int)c->ev0.size();
    // inside stream capture the record must be an EXTERNAL event-record node, or the event is owned by the graph and cannot be read from the host
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (timed) CKR(cudaStreamIsCapturing(st, &cap));
    const unsigned evflag = cap == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault;
    if (timed) CKR(cudaEventRecordWithFlags(c->ev0[row], st, evflag));
    if (uhc_env_step(c->eng, act_row, b->obs_cur, rew_row, c->d_cinfo, c->d_fail, c->d_end, c->d_pct, nullptr, st)) { g_ro_err = std::string("env step: ") + uhc_last_error(); return -1; }
    if (timed) CKR(cudaEventRecordWithFlags(c->ev1[row], st, evflag));
    n++;
    const bool eplog = b->ep_clip && b->ep_pct;
    k_rollout_post<<<(c->E + 255) / 256, 256, 0, st>>>(c->d_fail, c->d_end, mask_row, fail_row, mixed ? nullptr : exps_row, c->E, c->d_step, uhc_episode_log_dev(c->eng),
                                                       eplog ? b->ep_clip + (size_t)row * E : nullptr, eplog ? b->ep_pct + (size_t)row * E : nullptr,
                                                       eplog && b->ep_start ? b->ep_start + (size_t)row * E : nullptr);
    CKR(cudaGetLastError()); n++;
    return n;
}

}  // namespace

extern "C" {

const char *uhc_rollout_last_error(void) { return g_ro_err.c_str(); }

int uhc_rollout_set_step(UhcEngine *e, unsigned long long step) {
    if (!e) { g_ro_err = "uhc_rollout_set_step: null engine"; return -2; }
    RolloutCtx *c = ctx_of(e);
    if (!c->d_step) { CKR(cudaMalloc((void **)&c->d_step, sizeof(unsigned long long))); }
    CKR(cudaMemcpy(c->d_step, &step, sizeof step, cudaMemcpyHostToDevice));
    return 0;
}
int uhc_rollout_get_step(UhcEngine *e, unsigned long long *step) {
    if (!e || !step) { g_ro_err = "uhc_rollout_get_step: bad argument"; return -2; }
    RolloutCtx *c = ctx_of(e);
    *step = 0;
    if (c->d_step) { CKR(cudaDeviceSynchronize()); CKR(cudaMemcpy(step, c->d_step, sizeof *step, cudaMemcpyDeviceToHost)); }
    return 0;
}

static int make_policy(Policy *pol, const UhcMlp *mlp, const UhcMcp *mcp, UhcEngine *e, const char *who) {
    memset(pol, 0, sizeof *pol);
    if (mcp) {
        if (mcp->nprim < 1 || mcp->nprim > UHC_MCP_MAX_PRIM) { g_ro_err = std::string(who) + ": 1..8 primitives"; return -2; }
        pol->nprim = mcp->nprim;
        for (int k = 0; k < mcp->nprim; k++) pol->nets[k] = mcp->prim[k];
        pol->nets[mcp->nprim] = mcp->composer;
    } else pol->nets[0] = *mlp;
    const UhcMlp *m = &pol->nets[0];
    if (m->nlayers >= 1 && m->nlayers <= 8 && (m->dims[m->nlayers] != uhc_engine_act_dim(e) || m->dims[0] != uhc_engine_obs_dim(e))) {
        g_ro_err = std::string(who) + ": the policy's input / output widths are not the engine's obs / action dims"; return -2;
    }
    return 0;
}
static int policy_forward_impl(UhcEngine *e, const float *obs_dev, const Policy *pol, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                               unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                               void *stream) {
    RolloutCtx *c = ctx_of(e);
    int rc = ensure_scratch(c, pol);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (enqueue_policy(c, obs_dev, pol, zfilter_stats, zclip, update_filter, state_out_or_null, st) < 0) return -1;
    const UhcMlp *m = &pol->nets[0];
    k_gauss_sample_dev<<<(c->E + 7) / 8, 256, 0, st>>>(c->d_mean, log_std, mean_action_or_null, action_out, logp_out_or_null, c->E, m->dims[m->nlayers], seed, c->d_step);
    CKR(cudaGetLastError());
    return 0;
}
static int rollout_impl(UhcEngine *e, int T, int row0, const Policy *pol, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                        unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream) {
    RolloutCtx *c = ctx_of(e);
    int rc = ensure_scratch(c, pol);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (!use_graph) {
        for (int k = 0; k < T; k++) { const int n = enqueue_step(c, row0 + k, pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, st); if (n < 0) return -1; c->launches_per_step = n; }
        return 0;
    }
    GraphKey key; memset(&key, 0, sizeof key);
    key.T = T; key.row0 = row0; key.update_filter = update_filter; key.noise_rate = noise_rate; key.zclip = zclip; key.seed = seed; key.pol = *pol; key.buf = *buf;
    key.log_std = log_std; key.zstats = zfilter_stats; key.cur_gen = uhc::evalx::curriculum_gen(e);
    cudaGraphExec_t exec = nullptr;
    for (auto &g : c->graphs) if (g.first == key) { exec = g.second; break; }
    if (!exec) {
        // capture on a private stream (legacy-stream capture is not allowed), ordered after the caller's stream by an event
        cudaStream_t cs; CKR(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        cudaGraph_t graph = nullptr;
        CKR(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
        int n = 0;
        for (int k = 0; k < T && n >= 0; k++) n = enqueue_step(c, row0 + k, pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, cs);
        cudaError_t ce = cudaStreamEndCapture(cs, &graph);
        cudaStreamDestroy(cs);
        if (n < 0) { if (graph) cudaGraphDestroy(graph); return -1; }
        if (ce != cudaSuccess) { g_ro_err = std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce); return -1; }
        c->launches_per_step = n;
        CKR(cudaGraphInstantiate(&exec, graph, 0));
        cudaGraphDestroy(graph);
        if (c->graphs.size() >= 64) { cudaGraphExecDestroy(c->graphs.front().second); c->graphs.erase(c->graphs.begin()); }
        c->graphs.emplace_back(key, exec);
    }
    CKR(cudaGraphLaunch(exec, st));
    return 0;
}

int uhc_policy_forward(UhcEngine *e, const float *obs_dev, const UhcMlp *mlp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                       unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                       void *stream) {
    if (!e || !obs_dev || !mlp || !log_std || !zfilter_stats || !action_out) { g_ro_err = "uhc_policy_forward: bad argument"; return -2; }
    Policy pol; if (make_policy(&pol, mlp, nullptr, e, "uhc_policy_forward")) return -2;
    return policy_forward_impl(e, obs_dev, &pol, log_std, zfilter_stats, zclip, update_filter, seed, mean_action_or_null, state_out_or_null, action_out, logp_out_or_null, stream);
}
int uhc_policy_forward_mcp(UhcEngine *e, const float *obs_dev, const UhcMcp *mcp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                           unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                           void *stream) {
    if (!e || !obs_dev || !mcp || !log_std || !zfilter_stats || !action_out) { g_ro_err = "uhc_policy_forward_mcp: bad argument"; return -2; }
    Policy pol; if (make_policy(&pol, nullptr, mcp, e, "uhc_policy_forward_mcp")) return -2;
    return policy_forward_impl(e, obs_dev, &pol, log_std, zfilter_stats, zclip, update_filter, seed, mean_action_or_null, state_out_or_null, action_out, logp_out_or_null, stream);
}

int uhc_rollout(UhcEngine *e, int T, int row0, const UhcMlp *mlp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream) {
    if (!e || !mlp || !log_std || !zfilter_stats || !buf || T <= 0 || row0 < 0 || row0 + T > buf->T_cap) { g_ro_err = "uhc_rollout: bad argument"; return -2; }
    if (!buf->states || !buf->actions || !buf->rewards || !buf->masks || !buf->exps || !buf->obs_cur) { g_ro_err = "uhc_rollout: missing buffer"; return -2; }
    Policy pol; if (make_policy(&pol, mlp, nullptr, e, "uhc_rollout")) return -2;
    return rollout_impl(e, T, row0, &pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, use_graph, stream);
}
int uhc_rollout_mcp(UhcEngine *e, int T, int row0, const UhcMcp *mcp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                    unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream) {
    if (!e || !mcp || !log_std || !zfilter_stats || !buf || T <= 0 || row0 < 0 || row0 + T > buf->T_cap) { g_ro_err = "uhc_rollout_mcp: bad argument"; return -2; }
    if (!buf->states || !buf->actions || !buf->rewards || !buf->masks || !buf->exps || !buf->obs_cur) { g_ro_err = "uhc_rollout_mcp: missing buffer"; return -2; }
    Policy pol; if (make_policy(&pol, nullptr, mcp, e, "uhc_rollout_mcp")) return -2;
    return rollout_impl(e, T, row0, &pol, log_std, zfilter_stats, zclip, update_filter, seed, noise_rate, buf, use_graph, stream);
}

// events around the env-step kernel of rows 0 .. nrows-1 (recorded on the launching stream, also inside graph replays); 0 disables.
// Changing it drops the cached graphs.
int uhc_rollout_time_env_step(UhcEngine *e, int nrows) {
    if (!e || nrows < 0) { g_ro_err = "uhc_rollout_time_env_step: bad argument"; return -2; }
    RolloutCtx *c = ctx_of(e);
    CKR(cudaDeviceSynchronize());
    for (auto &g : c->graphs) cudaGraphExecDestroy(g.second);
    c->graphs.clear();
    for (cudaEvent_t ev : c->ev0) cudaEventDestroy(ev);
    for (cudaEvent_t ev : c->ev1) cudaEventDestroy(ev);
    c->ev0.assign(nrows, nullptr); c->ev1.assign(nrows, nullptr);
    for (int i = 0; i < nrows; i++) { CKR(cudaEventCreate(&c->ev0[i])); CKR(cudaEventCreate(&c->ev1[i])); }
    return 0;
}
int uhc_rollout_env_step_ms(UhcEngine *e, int row, float *ms) {
    if (!e || !ms) { g_ro_err = "uhc_rollout_env_step_ms: bad argument"; return -2; }
    RolloutCtx *c = ctx_of(e);
    if (row < 0 || row >= (int)c->ev0.size()) { g_ro_err = "uhc_rollout_env_step_ms: row not timed"; return -2; }
    CKR(cudaEventSynchronize(c->ev1[row]));
    CKR(cudaEventElapsedTime(ms, c->ev0[row], c->ev1[row]));
    return 0;
}

int uhc_rollout_launches_per_step(UhcEngine *e) { return e ? ctx_of(e)->launches_per_step : -1; }

void uhc_rollout_release(UhcEngine *e) {   // called by the binding before uhc_engine_destroy
    for (size_t i = 0; i < g_ctx.size(); i++) if (g_ctx[i]->eng == e) {
        RolloutCtx *c = g_ctx[i];
        for (auto &g : c->graphs) cudaGraphExecDestroy(g.second);
        for (cudaEvent_t ev : c->ev0) cudaEventDestroy(ev);
        for (cudaEvent_t ev : c->ev1) cudaEventDestroy(ev);
        for (auto &nsj : c->ns) for (void *p : nsj.acts) if (p) cudaFree(p);
        for (void *p : {(void *)c->d_xall, (void *)c->d_comp, (void *)c->d_zws, (void *)c->d_step, (void *)c->d_mean, (void *)c->d_mean_action, (void *)c->d_cinfo, (void *)c->d_pct, (void *)c->d_fail, (void *)c->d_end}) if (p) cudaFree(p);
        delete c; g_ctx.erase(g_ctx.begin() + i); return;
    }
}

}  // extern "C"

// ---- the policy forward of the device evaluation (eval_glue.h): the kernels of uhc_policy_forward(_mcp), enqueued from eval.cu's graphs
namespace uhc {
namespace evalx {

int policy_prepare(UhcEngine *e, const UhcMlp *mlp, const UhcMcp *mcp, unsigned long long *gen, std::string *err) {
    Policy pol;
    if (make_policy(&pol, mlp, mcp, e, mcp ? "uhc_eval_run_mcp" : "uhc_eval_run")) { *err = g_ro_err; return -2; }
    RolloutCtx *c = ctx_of(e);
    const int rc = ensure_scratch(c, &pol);
    if (rc) { *err = g_ro_err; return rc; }
    *gen = c->scratch_gen;
    return 0;
}

int policy_enqueue(UhcEngine *e, const UhcMlp *mlp, const UhcMcp *mcp, const float *obs, const float *log_std, double *zstats, float zclip,
                   const unsigned char *mean_action, float *action, cudaStream_t st, std::string *err) {
    Policy pol;
    if (make_policy(&pol, mlp, mcp, e, "uhc_eval_run")) { *err = g_ro_err; return -2; }
    RolloutCtx *c = ctx_of(e);
    if (enqueue_policy(c, obs, &pol, zstats, zclip, 0, nullptr, st) < 0) { *err = g_ro_err; return -1; }
    const UhcMlp *m = &pol.nets[0];
    k_gauss_sample_dev<<<(c->E + 7) / 8, 256, 0, st>>>(c->d_mean, log_std, mean_action, action, nullptr, c->E, m->dims[m->nlayers], 0, c->d_step);
    const cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) { *err = std::string("k_gauss_sample_dev: ") + cudaGetErrorString(ce); return -1; }
    return 0;
}

// ---- the grouped policy forward of uhc_eval_run_groups: G policies of one architecture over consecutive row ranges, with scratch of its
// own (the rollout's ns[] / d_mean pointers are baked into its graphs and the single-policy evaluation's)
namespace {
struct GroupCtx {
    UhcEngine *eng = nullptr; int E = 0;
    RolloutCtx::NetScratch ns[UHC_MCP_MAX_PRIM + 1];
    float *d_mean = nullptr; int mean_cap = 0;
    float *d_xall = nullptr, *d_comp = nullptr; size_t xall_cap = 0;
    float *d_log_std0 = nullptr; int ls_cap = 0;   // zeros: with the all-ones mask k_gauss_sample_dev then writes mean + 1 * 0, what any finite log_std gives
    unsigned long long *d_step = nullptr;          // read (not used) by the deterministic sampler
    unsigned long long gen = 0;                    // bumped whenever the scratch above is reallocated
};
std::vector<GroupCtx *> g_gctx;

GroupCtx *gctx_of(UhcEngine *e) {
    for (GroupCtx *c : g_gctx) if (c->eng == e) return c;
    GroupCtx *c = new GroupCtx(); c->eng = e; c->E = uhc_num_envs(e);
    g_gctx.push_back(c);
    return c;
}

// the checks ensure_scratch makes, without allocating
int check_policy(const Policy *pol) {
    const int P = pol->nprim, nnets = P > 0 ? P + 1 : 1;
    const UhcMlp *m0 = &pol->nets[0];
    for (int j = 0; j < nnets; j++) {
        const UhcMlp *m = &pol->nets[j];
        if (m->nlayers < 1 || m->nlayers > 8) { g_ro_err = "UhcMlp: 1..8 layers"; return -2; }
        if (m->dims[0] != m0->dims[0]) { g_ro_err = "UhcMcp: every net reads the same observation"; return -2; }
        if (j < P && m->dims[m->nlayers] != m0->dims[m0->nlayers]) { g_ro_err = "UhcMcp: the primitives must share the action width"; return -2; }
        if (P > 0 && j == P && m->dims[m->nlayers] != P) { g_ro_err = "UhcMcp: the composer's output width must be the number of primitives"; return -2; }
        for (int i = 0; i < m->nlayers; i++) {
            if (m->kp[i] != pad64(m->dims[i])) { g_ro_err = "UhcMlp: kp[i] must be dims[i] rounded up to 64"; return -2; }
            if (!m->W_bf16[i]) { g_ro_err = "UhcMlp: null weights"; return -2; }
        }
    }
    return 0;
}
// every group's policy must have group 0's architecture: primitive count, and per net the layer count, activation, widths and K padding
bool same_arch(const Policy *a, const Policy *b) {
    if (a->nprim != b->nprim) return false;
    for (int j = 0; j < (a->nprim > 0 ? a->nprim + 1 : 1); j++) {
        const UhcMlp &x = a->nets[j], &y = b->nets[j];
        if (x.nlayers != y.nlayers || x.act != y.act) return false;
        for (int i = 0; i <= x.nlayers; i++) if (x.dims[i] != y.dims[i]) return false;
        for (int i = 0; i < x.nlayers; i++) if (x.kp[i] != y.kp[i]) return false;
    }
    return true;
}
int make_group_policies(UhcEngine *e, int G, const UhcMlp *mlps, const UhcMcp *mcps, std::vector<Policy> *pols) {
    const char *who = mcps ? "uhc_eval_run_groups_mcp" : "uhc_eval_run_groups";
    pols->resize(G);
    for (int g = 0; g < G; g++) {
        if (make_policy(&(*pols)[g], mlps ? mlps + g : nullptr, mcps ? mcps + g : nullptr, e, who)) return -2;
        if (check_policy(&(*pols)[g])) { g_ro_err = std::string(who) + ": " + g_ro_err; return -2; }
        if (g > 0 && !same_arch(&(*pols)[0], &(*pols)[g])) { g_ro_err = std::string(who) + ": every group's policy must have the same layer widths, K padding, activation and primitive count"; return -2; }
    }
    return 0;
}
int ensure_group_scratch(GroupCtx *c, const Policy *pol) {
    const size_t E = c->E;
    const int P = pol->nprim;
    const UhcMlp *m0 = &pol->nets[0];
    const int A = m0->dims[m0->nlayers];
    if (!c->d_step) { CKR(cudaMalloc((void **)&c->d_step, sizeof(unsigned long long))); CKR(cudaMemset(c->d_step, 0, sizeof(unsigned long long))); }
    for (int j = 0; j < (P > 0 ? P + 1 : 1); j++) {
        const UhcMlp *m = &pol->nets[j];
        for (int i = 0; i < m->nlayers; i++) {
            if (i == 0 && j > 0) continue;       // the normalised observation feeds every net
            const int ld = m->kp[i];
            if (c->ns[j].ld[i] != ld) {
                if (c->ns[j].acts[i]) cudaFree(c->ns[j].acts[i]);
                CKR(cudaMalloc(&c->ns[j].acts[i], E * ld * 2)); CKR(cudaMemset(c->ns[j].acts[i], 0, E * ld * 2));
                c->ns[j].ld[i] = ld; c->gen++;
            }
        }
    }
    if (c->mean_cap < A) {
        if (c->d_mean) cudaFree(c->d_mean);
        if (c->d_log_std0) cudaFree(c->d_log_std0);
        CKR(cudaMalloc((void **)&c->d_mean, E * A * 4)); CKR(cudaMemset(c->d_mean, 0, E * A * 4));
        CKR(cudaMalloc((void **)&c->d_log_std0, A * 4)); CKR(cudaMemset(c->d_log_std0, 0, A * 4));
        c->mean_cap = A; c->gen++;
    }
    if (P > 0 && c->xall_cap < (size_t)P * E * A) {
        if (c->d_xall) cudaFree(c->d_xall);
        if (c->d_comp) cudaFree(c->d_comp);
        CKR(cudaMalloc((void **)&c->d_xall, (size_t)P * E * A * 4)); CKR(cudaMemset(c->d_xall, 0, (size_t)P * E * A * 4));
        CKR(cudaMalloc((void **)&c->d_comp, E * UHC_MCP_MAX_PRIM * 4)); CKR(cudaMemset(c->d_comp, 0, E * UHC_MCP_MAX_PRIM * 4));
        c->xall_cap = (size_t)P * E * A; c->gen++;
    }
    return 0;
}
}  // namespace

int groups_prepare(UhcEngine *e, int G, const UhcMlp *mlps, const UhcMcp *mcps, unsigned long long *gen, std::string *err) {
    std::vector<Policy> pols;
    if (make_group_policies(e, G, mlps, mcps, &pols)) { *err = g_ro_err; return -2; }
    GroupCtx *c = gctx_of(e);
    const int rc = ensure_group_scratch(c, &pols[0]);
    if (rc) { *err = g_ro_err; return rc; }
    *gen = c->gen;
    return 0;
}

int groups_enqueue(UhcEngine *e, int G, const int *row0, const UhcMlp *mlps, const UhcMcp *mcps, const double *const *zstats, float zclip, const float *obs,
                   const unsigned char *mean_action, float *action, cudaStream_t st, std::string *err) {
    std::vector<Policy> pols;
    if (make_group_policies(e, G, mlps, mcps, &pols)) { *err = g_ro_err; return -2; }
    GroupCtx *c = gctx_of(e);
    const Policy &p0 = pols[0];
    const UhcMlp *m0 = &p0.nets[0];
    const int E = c->E, D = m0->dims[0], P = p0.nprim, A = m0->dims[m0->nlayers], ntot = row0[G];
    ZGroups zg;
    memset(&zg, 0, sizeof zg);
    zg.G = G;
    std::vector<int> rows(G);
    for (int g = 0; g <= G; g++) zg.row0[g] = row0[g];
    for (int g = 0; g < G; g++) { zg.stats[g] = zstats[g]; rows[g] = row0[g + 1] - row0[g]; }
    k_zfilter_apply_bf16_grouped<<<1056, 256, 0, st>>>(obs, nullptr, (unsigned short *)c->ns[0].acts[0], ntot, D, m0->kp[0], zg, zclip);
    cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) { *err = std::string("k_zfilter_apply_bf16_grouped: ") + cudaGetErrorString(ce); return -1; }
    std::vector<const void *> W(G);
    std::vector<const float *> b(G);
    for (int j = 0; j < (P > 0 ? P + 1 : 1); j++) {
        const UhcMlp *m = &p0.nets[j];
        const bool composer = P > 0 && j == P;
        float *out = P == 0 ? c->d_mean : (composer ? c->d_comp : c->d_xall + (size_t)j * E * A);
        for (int i = 0; i < m->nlayers; i++) {
            const bool last = i == m->nlayers - 1;
            const void *in = i == 0 ? c->ns[0].acts[0] : c->ns[j].acts[i];
            for (int g = 0; g < G; g++) { W[g] = pols[g].nets[j].W_bf16[i]; b[g] = pols[g].nets[j].bias[i]; }
            if (uhc_linear_forward_tc_grouped(G, row0, rows.data(), in, W.data(), b.data(), last ? nullptr : c->ns[j].acts[i + 1], last ? out : nullptr, E,
                                              m->dims[i + 1], m->kp[i], last ? 0 : c->ns[j].ld[i + 1], (last && !composer) ? UHC_ACT_NONE : m->act, st)) {
                *err = std::string("grouped policy GEMM: ") + uhc_tc_last_error(); return -1;
            }
        }
    }
    // the mixture head is row-wise: run over every row (rows past the groups hold zeros or earlier values and are never read)
    if (P > 0 && uhc_mcp_combine(c->d_xall, c->d_comp, nullptr, c->d_mean, E, A, P, st)) { *err = std::string("mixture head: ") + uhc_nn_last_error(); return -1; }
    k_gauss_sample_dev<<<(ntot + 7) / 8, 256, 0, st>>>(c->d_mean, c->d_log_std0, mean_action, action, nullptr, ntot, A, 0, c->d_step);
    ce = cudaGetLastError();
    if (ce != cudaSuccess) { *err = std::string("k_gauss_sample_dev: ") + cudaGetErrorString(ce); return -1; }
    return 0;
}

void groups_release(UhcEngine *e) {
    for (size_t i = 0; i < g_gctx.size(); i++) if (g_gctx[i]->eng == e) {
        GroupCtx *c = g_gctx[i];
        for (auto &nsj : c->ns) for (void *p : nsj.acts) if (p) cudaFree(p);
        for (void *p : {(void *)c->d_mean, (void *)c->d_xall, (void *)c->d_comp, (void *)c->d_log_std0, (void *)c->d_step}) if (p) cudaFree(p);
        delete c; g_gctx.erase(g_gctx.begin() + i); return;
    }
}

}  // namespace evalx
}  // namespace uhc
