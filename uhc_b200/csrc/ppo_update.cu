// ppo_update.cu -- uhc_ppo_update (include/uhc_ppo.h): one PPO iteration's whole update behind a single C-ABI call.
//
// Replaces the reference's Python  AgentPG.update_params -> estimate_advantages -> AgentPPO.update_policy
// (uhc/khrylib/rl/agents/agent_pg.py:39-56, core/common.py:5-25, agents/agent_ppo.py:16-65) and the torch autograd / Adam work under it by
//   k_f32_to_bf16_padded, k_transpose_bf16     states -> bf16 K-padded operand and its transpose (once per update)
//   k_linear_tc                                every GEMM: forward (bias + activation fused, fp32 pre-activations kept), dX = dZ W, dW = dZ^T X
//   k_gae, k_moments, k_normalize              GAE with V(s_T) bootstrap, advantage normalisation over the GLOBAL batch
//   k_value_grad, k_ppo_grad                   loss gradients wrt the heads (pre-scaled by the global row counts)
//   k_dact_bf16                                dz = dh act'(z) -> bf16 dz, dz^T and the bias gradient in one pass
//   k_sqsum, k_adam                            clip_grad_norm_ scale + torch.optim.Adam, one launch per net on the flat tensors
//   ncclAllReduce                              the one collective: each net's flat gradient tensor, on a side stream under the other net's work;
//                                              the statistics tail (k_stats_pack / k_stats_join) and uhc_ppo_update_ex's extra payload ride the first one
// Per epoch the order is value forward/backward -> value all-reduce starts -> policy forward/gradient/backward -> policy all-reduce starts ->
// value Adam -> policy Adam: the two nets are independent inside an epoch, so this equals the reference's "value step, then policy step".
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/uhc_nn.h"
#include "../../include/uhc_ppo.h"
#include "errors.h"

namespace {
thread_local long g_launches = 0;      // kernels enqueued by the current uhc_ppo_update call (every CKU call below launches exactly one)
#define CKU(x, what) do { ++g_launches; if ((x) != 0) return uhc_err_prefix(what); } while (0)

inline long pad64(long n) { return (n + 63) / 64 * 64; }

// ---- exact fp64 statistics through an fp32 all-reduce(sum): base-2^18 fixed-point digit planes (5 planes: |x| < 2^60, lsb 2^-30); every
// digit is an integer below 2^18 in magnitude, so the fp32 sum over up to 32 ranks is exact.
constexpr int PLANES = 5, PLANE_BITS = 18, PLANE_TOP = 60;
// d = [adv sum, adv sum of squares, rows, selected rows, ZFilter increment in additive form (n, sum, sum of squares) since the last agreement]
__global__ void k_stats_pack(const double *__restrict__ mom2, double rows, const double *__restrict__ cnt, const double *__restrict__ zstats,
                             const double *__restrict__ zsync, int D, float *__restrict__ planes) {
    const int nd = 4 + 1 + 2 * D;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nd) return;
    double x;
    if (i < 2) x = mom2[i];
    else if (i == 2) x = rows;
    else if (i == 3) x = cnt[0];
    else {
        const int j = i - 4;
        const double n = zstats[0];
        double s;
        if (j == 0) s = n;
        else if (j <= D) s = n * zstats[j];
        else { const double mean = zstats[j - D]; s = zstats[j] + n * mean * mean; }
        x = s - zsync[j];
    }
    double r = x;
    for (int k = 0; k < PLANES; ++k) {
        const double scale = exp2((double)(PLANE_TOP - PLANE_BITS * (k + 1)));
        const double c = trunc(r / scale);
        r -= c * scale;
        planes[(size_t)k * nd + i] = (float)c;
    }
}
// after the all-reduce: global advantage moments / row count / 1 / selected rows; zsync += the ranks' increments
__global__ void k_stats_join(const float *__restrict__ planes, int D, double *__restrict__ mom2, double *__restrict__ ntot, float *__restrict__ inv_count,
                             double *__restrict__ zsync) {
    const int nd = 4 + 1 + 2 * D;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nd) return;
    double g = 0.0;
    for (int k = 0; k < PLANES; ++k) g += (double)planes[(size_t)k * nd + i] * exp2((double)(PLANE_TOP - PLANE_BITS * (k + 1)));
    if (i < 2) mom2[i] = g;
    else if (i == 2) ntot[0] = g;
    else if (i == 3) inv_count[0] = (float)(1.0 / (g < 1.0 ? 1.0 : g));
    else zsync[i - 4] += g;
}
// additive form -> (n, mean, S): every rank ends with the same running statistics
__global__ void k_zfilter_from_sums(const double *__restrict__ zsync, int D, double *__restrict__ zstats) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > 2 * D) return;
    const double n = zsync[0];
    if (j == 0) { zstats[0] = n; return; }
    const int d = j <= D ? j : j - D;
    const double mean = zsync[d] / (n < 1.0 ? 1.0 : n);
    if (j <= D) zstats[j] = mean;
    else { const double S = zsync[j] - n * mean * mean; zstats[j] = S < 0.0 ? 0.0 : S; }
}
__global__ void k_count_selected(const float *__restrict__ exps, size_t n, double *__restrict__ out) {
    __shared__ double sh[256];
    double s = 0.0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) s += exps[i] != 0.f ? 1.0 : 0.0;
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) atomicAdd(out, sh[0]);
}
__global__ void k_inv_count(const double *__restrict__ cnt, float *__restrict__ inv) { const double c = cnt[0]; inv[0] = (float)(1.0 / (c < 1.0 ? 1.0 : c)); }

// ---- NCCL without a link-time dependency: the process that hands us an ncclComm_t has libnccl loaded already
UhcAllReduceFn nccl_all_reduce() {
    static const UhcAllReduceFn fn = [] {       // a function-local static: one lookup, however many threads update at once
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        return h ? (UhcAllReduceFn)dlsym(h, "ncclAllReduce") : (UhcAllReduceFn) nullptr;
    }();
    return fn;
}
constexpr int NCCL_FLOAT32 = 7, NCCL_SUM = 0;

struct NetBuf { void *acts[9] = {nullptr}; void *actsT[9] = {nullptr}; float *z[8] = {nullptr}; float *out = nullptr; };   // actsT[i]: [dims[i]][rows rounded up to 64] bf16, written by the forward epilogue
}  // namespace

struct UhcPpoTrainer {
    int device = 0; long cap = 0; int cap_envs = 0;
    std::vector<UhcNetDesc> pnets;     // the policy: one MLP (nprim = 0) or nprim primitives followed by the composer (PolicyMCP); all share pnets[0]'s flat storage
    std::vector<NetBuf> pbufs;
    int nprim = 0;
    float *xall = nullptr, *mixw = nullptr, *dxall = nullptr, *dcomp = nullptr, *mean = nullptr;   // PolicyMCP: primitive outputs [P][M][A], softmax weights [M][P], their gradients, the mixture mean
    UhcNetDesc val{};
    NetBuf vb;
    void *xb = nullptr, *xT = nullptr, *lb = nullptr;                   // bf16 states [M][Dp], transpose [D][Mp], last states [E][Dp]
    float *dWpad = nullptr; long dWpad_n = 0;                          // dW of a layer whose input width is not a multiple of 4, at a pitch the TMA engine accepts
    void *dz2 = nullptr, *dzT2 = nullptr;                               // second dz / dz^T pair: the fused dX + activation-backward GEMM reads one pair and writes the other
    void *dz = nullptr, *dzT = nullptr, *hT = nullptr, *WT = nullptr;   // shared backward scratch (the nets run back to back on one stream)
    float *dh = nullptr, *dmean = nullptr, *dv = nullptr, *fixed = nullptr, *adv = nullptr, *ret = nullptr, *last_v = nullptr, *inv_count = nullptr;
    double *mom = nullptr, *cnt = nullptr, *ntot = nullptr, *sq = nullptr;
    cudaStream_t side = nullptr;
    cudaEvent_t ev_ready = nullptr, ev_v = nullptr, ev_p = nullptr;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timing; size_t timing_used = 0;
    long comm_bytes = 0; int comm_calls = 0;
    UhcAllReduceFn all_reduce = nullptr;     // uhc_ppo_trainer_set_all_reduce; nullptr = ncclAllReduce
    long launches = 0;
    std::vector<void *> allocs;
};

namespace {
int check_net(const UhcNetDesc &n, const char *name) {
    if (n.nlayers < 1 || n.nlayers > 8 || !n.flat || !n.gfull || !n.adam_m || !n.adam_v) { uhc_err() = std::string(name) + ": bad UhcNetDesc"; return -2; }
    for (int i = 0; i < n.nlayers; i++)
        if (n.dims[i] <= 0 || n.dims[i + 1] <= 0 || n.kp[i] != pad64(n.dims[i]) || !n.W_bf16[i]) { uhc_err() = std::string(name) + ": kp[i] must be dims[i] rounded up to 64 and W_bf16[i] set"; return -2; }
    return 0;
}
template <class T> int dalloc(UhcPpoTrainer *t, T **p, size_t bytes, bool zero) {
    CK(cudaMalloc((void **)p, bytes ? bytes : 16));
    t->allocs.push_back((void *)*p);
    if (zero) CK(cudaMemset(*p, 0, bytes ? bytes : 16));
    return 0;
}
int alloc_net(UhcPpoTrainer *t, const UhcNetDesc &n, NetBuf &nb, long cap, bool own_out) {
    for (int i = 0; i < n.nlayers - 1; i++) {
        if (dalloc(t, &nb.acts[i + 1], (size_t)cap * pad64(n.dims[i + 1]) * 2, true)) return -1;    // bf16, zero padded once (the GEMMs write the first N columns)
        if (uhc_tc_tma_store_enabled() && dalloc(t, &nb.actsT[i + 1], (size_t)n.dims[i + 1] * pad64(cap) * 2, true)) return -1;
        if (dalloc(t, &nb.z[i], (size_t)cap * n.dims[i + 1] * 4, false)) return -1;
    }
    if (n.head_act != UHC_ACT_NONE && dalloc(t, &nb.z[n.nlayers - 1], (size_t)cap * n.dims[n.nlayers] * 4, false)) return -1;   // activated output layer (MCP composer)
    return own_out ? dalloc(t, &nb.out, (size_t)cap * n.dims[n.nlayers] * 4, false) : 0;
}
// forward keeping what the backward pass needs (bf16 activations, fp32 pre-activations); train = false: plain inference chain on `rows` rows
int net_forward(const UhcNetDesc &n, NetBuf &nb, const void *x, long rows, bool train, cudaStream_t st) {
    const void *h = x;
    for (int i = 0; i < n.nlayers; i++) {
        const bool last = i == n.nlayers - 1;
        const int N = n.dims[i + 1];
        const int act = last ? n.head_act : n.act;
        if (train && !last && nb.actsT[i + 1]) {      // hidden layer of a training forward: the epilogue also writes the transposed activation the dW GEMM needs
            CKU(uhc_linear_forward_tc_train_t(h, n.W_bf16[i], n.flat + n.b_off[i], nb.acts[i + 1], nb.actsT[i + 1], (int)pad64(rows), act == UHC_ACT_NONE ? nullptr : nb.z[i],
                                              (int)rows, N, n.kp[i], (int)pad64(N), act, st), "forward GEMM");
            h = nb.acts[i + 1];
            continue;
        }
        CKU(uhc_linear_forward_tc_train(h, n.W_bf16[i], n.flat + n.b_off[i], last ? nullptr : nb.acts[i + 1], last ? nb.out : nullptr,
                                        (!train || act == UHC_ACT_NONE) ? nullptr : nb.z[i], (int)rows, N, n.kp[i], last ? 0 : (int)pad64(N), act, st), "forward GEMM");
        h = nb.acts[i + 1];
    }
    return 0;
}
// dW / db straight into the flat gradient tensor
int net_backward(UhcPpoTrainer *t, const UhcNetDesc &n, NetBuf &nb, const float *dy, long M, cudaStream_t st) {
    const long Mp = pad64(M);
    const float *dh = dy;
    void *dz = t->dz, *dzT = t->dzT, *dz_o = t->dz2, *dzT_o = t->dzT2;
    bool have_dz = false;        // dz / dz^T / db of this layer were already produced by the layer above's fused dX GEMM
    for (int i = n.nlayers - 1; i >= 0; --i) {
        const int N = n.dims[i + 1], K = n.dims[i];
        const long Np = pad64(N);
        const int act = i < n.nlayers - 1 ? n.act : n.head_act;
        if (!have_dz)
            CKU(uhc_dact_bf16(dh, act != UHC_ACT_NONE ? nb.z[i] : nullptr, dz, dzT, n.gfull + n.b_off[i], (int)M, N, (int)Np, (int)Mp, act, st), "activation backward");
        have_dz = false;
        const void *hT = t->xT;
        if (i > 0) {
            if (nb.actsT[i]) hT = nb.actsT[i];           // written by the forward pass' epilogue with pitch pad64(M)
            else { CKU(uhc_transpose_bf16(nb.acts[i], t->hT, (int)M, K, (int)pad64(K), (int)Mp, st), "transpose h"); hT = t->hT; }
        }
        // dW = dz^T h.  A row length that is not a multiple of 4 floats (657 inputs) has no tensor map: that product runs at a padded pitch, then the rows are copied
        const int Kq = (K + 3) & ~3;
        if (K != Kq && t->dWpad && (long)N * Kq <= t->dWpad_n && uhc_linear_forward_tc_f32_pitched(dzT, hT, t->dWpad, Kq, N, K, (int)Mp, st) == 0) {
            g_launches += 2;          // the GEMM and the row copy
            CK(cudaMemcpy2DAsync(n.gfull + n.w_off[i], (size_t)K * 4, t->dWpad, (size_t)Kq * 4, (size_t)K * 4, N, cudaMemcpyDeviceToDevice, st));
        } else
            CKU(uhc_linear_forward_tc(dzT, hT, nullptr, nullptr, n.gfull + n.w_off[i], N, K, (int)Mp, 0, UHC_ACT_NONE, st), "dW GEMM");
        if (i > 0) {
            CKU(uhc_transpose_bf16(n.W_bf16[i], t->WT, N, K, n.kp[i], (int)Np, st), "transpose W");
            if (uhc_tc_tma_store_enabled() && n.act != UHC_ACT_NONE && K % 4 == 0) {
                // dz_prev = (dz W) * act'(z_prev) with its transpose and the bias gradient, all from the GEMM's epilogue
                CKU(uhc_linear_dx_dact_tc(dz, t->WT, nb.z[i - 1], dz_o, dzT_o, n.gfull + n.b_off[i - 1], (int)M, K, (int)Np, (int)pad64(K), (int)Mp, n.act, st), "dX + activation backward GEMM");
                void *s1 = dz; dz = dz_o; dz_o = s1; s1 = dzT; dzT = dzT_o; dzT_o = s1;
                have_dz = true;
            } else {
                CKU(uhc_linear_forward_tc(dz, t->WT, nullptr, nullptr, t->dh, (int)M, K, (int)Np, 0, UHC_ACT_NONE, st), "dX GEMM");                  // dh_prev = dz W
                dh = t->dh;
            }
        }
    }
    return 0;
}
int refresh_bf16(const UhcNetDesc &n, cudaStream_t st) {
    for (int i = 0; i < n.nlayers; i++) CKU(uhc_f32_to_bf16_padded(n.flat + n.w_off[i], n.W_bf16[i], n.dims[i + 1], n.dims[i], n.kp[i], st), "bf16 weight refresh");
    return 0;
}
// the policy's mean for every row: the single MLP's output, or the PolicyMCP mixture (policy_mcp.py:28-36)
int policy_forward(UhcPpoTrainer *t, long M, const float **mean_out, cudaStream_t st) {
    const int P = t->nprim, A = t->pnets[0].dims[t->pnets[0].nlayers];
    for (int k = 0; k < P; k++) t->pbufs[k].out = t->xall + (size_t)k * M * A;       // [P][M][A], contiguous for this M
    for (size_t j = 0; j < t->pnets.size(); j++) if (net_forward(t->pnets[j], t->pbufs[j], t->xb, M, true, st)) return -1;
    if (P == 0) { *mean_out = t->pbufs[0].out; return 0; }
    CKU(uhc_mcp_combine(t->xall, t->pbufs[P].out, t->mixw, t->mean, (int)M, A, P, st), "mixture head");
    *mean_out = t->mean;
    return 0;
}
int policy_backward(UhcPpoTrainer *t, const float *dmean, long M, cudaStream_t st) {
    const int P = t->nprim, A = t->pnets[0].dims[t->pnets[0].nlayers];
    if (P == 0) return net_backward(t, t->pnets[0], t->pbufs[0], dmean, M, st);
    CKU(uhc_mcp_backward(t->xall, t->mixw, dmean, t->dxall, t->dcomp, (int)M, A, P, st), "mixture head backward");
    for (int k = 0; k < P; k++) if (net_backward(t, t->pnets[k], t->pbufs[k], t->dxall + (size_t)k * M * A, M, st)) return -1;
    return net_backward(t, t->pnets[P], t->pbufs[P], t->dcomp, M, st);
}
int start_all_reduce(UhcPpoTrainer *t, void *comm, float *buf, size_t n, cudaEvent_t done, cudaStream_t st) {
    const UhcAllReduceFn ar = t->all_reduce ? t->all_reduce : nccl_all_reduce();
    if (!ar) { uhc_err() = "uhc_ppo_update: an ncclComm_t was passed but libnccl.so.2 / ncclAllReduce cannot be resolved"; return -1; }
    CK(cudaEventRecord(t->ev_ready, st));
    CK(cudaStreamWaitEvent(t->side, t->ev_ready, 0));
    if (t->timing_used == t->timing.size()) {
        cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
        t->timing.push_back({a, b});
    }
    auto &tm = t->timing[t->timing_used++];
    CK(cudaEventRecord(tm.first, t->side));
    const int rc = ar(buf, buf, n, NCCL_FLOAT32, NCCL_SUM, comm, (void *)t->side);
    if (rc != 0) {
        --t->timing_used;     // its end event was never recorded: uhc_ppo_comm_stats must not read the pair
        uhc_err() = std::string("the gradient all-reduce (") + (t->all_reduce ? "the installed collective" : "ncclAllReduce") + ") failed with code " + std::to_string(rc);
        return -1;
    }
    CK(cudaEventRecord(tm.second, t->side));
    CK(cudaEventRecord(done, t->side));
    t->comm_bytes += (long)(n * sizeof(float)); t->comm_calls++;
    return 0;
}
}  // namespace

// the PPO epochs on t->xb / t->xT / t->adv / t->ret: per epoch one value step then one clipped-surrogate policy step (agent_ppo.py:46-51), see the file header
// for the order of the collectives.  stats_tail: the first value all-reduce carries the statistics planes (uhc_ppo_update with world > 1), and
// n_extra caller floats behind them, whose sum over the ranks goes to extra_out.
static int run_epochs(UhcPpoTrainer *t, const float *actions, const float *exps, const float *log_std, long M, const UhcPpoCfg *cfg, int *adam_step_policy,
                      int *adam_step_value, int *policy_steps_done, double *zfilter_stats, double *zfilter_sync, void *comm, int world, bool stats_tail,
                      long n_extra, float *extra_out, bool value_forward_done, float *losses_out, cudaStream_t st) {
    const UhcNetDesc &pol = t->pnets[0], &val = t->val;
    const int D = pol.dims[0], A = pol.dims[pol.nlayers];
    const int nd = 4 + 1 + 2 * D;
    float *tail = val.gfull + val.nflat;
    // ---- old-policy mean: the fixed log-probabilities and epoch 0's policy forward (same weights)
    const float *pmean = nullptr;
    if (policy_forward(t, M, &pmean, st)) return -1;
    CKU(uhc_gaussian_logprob(pmean, log_std, actions, t->fixed, (int)M, A, st), "fixed log-probabilities");

    for (int ep = 0; ep < cfg->epochs; ++ep) {
        if ((ep > 0 || !value_forward_done) && net_forward(val, t->vb, t->xb, M, true, st)) return -1;
        CK(cudaMemsetAsync(losses_out, 0, 2 * sizeof(float), st));
        CKU(uhc_value_grad_n(t->vb.out, t->ret, t->dv, losses_out + 1, (int)M, M * world, st), "value gradient");
        if (net_backward(t, val, t->vb, t->dv, M, st)) return -1;
        const bool with_tail = stats_tail && ep == 0;
        if (comm && start_all_reduce(t, comm, val.gfull, (size_t)val.nflat + (with_tail ? (size_t)PLANES * nd + n_extra : 0), t->ev_v, st)) return -1;
        if (with_tail) {    // the global statistics are needed before the first policy gradient
            CK(cudaStreamWaitEvent(st, t->ev_v, 0));
            ++g_launches; k_stats_join<<<(nd + 255) / 256, 256, 0, st>>>(tail, D, t->mom, t->ntot, t->inv_count, zfilter_sync); CK(cudaGetLastError());
            CKU(uhc_adv_normalize(t->adv, M, t->mom, t->ntot, st), "advantage normalisation (global)");
            ++g_launches; k_zfilter_from_sums<<<(2 * D + 1 + 255) / 256, 256, 0, st>>>(zfilter_sync, D, zfilter_stats); CK(cudaGetLastError());
            if (n_extra) CK(cudaMemcpyAsync(extra_out, tail + (size_t)PLANES * nd, (size_t)n_extra * sizeof(float), cudaMemcpyDeviceToDevice, st));
        }
        if (ep > 0 && policy_forward(t, M, &pmean, st)) return -1;
        CKU(uhc_ppo_policy_grad_dev(pmean, log_std, actions, t->adv, t->fixed, exps, cfg->clip_eps, t->inv_count, t->dmean, losses_out, (int)M, A, st), "policy gradient");
        if (policy_backward(t, t->dmean, M, st)) return -1;
        if (comm && start_all_reduce(t, comm, pol.gfull, (size_t)pol.nflat, t->ev_p, st)) return -1;
        // value step first, as the reference; the policy collective is still in flight
        if (comm) CK(cudaStreamWaitEvent(st, t->ev_v, 0));
        *adam_step_value += 1;
        CKU(uhc_adam_step(val.flat, val.gfull, val.adam_m, val.adam_v, val.nflat, val.lr, 0.9f, 0.999f, 1e-8f, *adam_step_value, nullptr, 0.f, st), "value Adam");
        if (refresh_bf16(val, st)) return -1;
        if (comm) CK(cudaStreamWaitEvent(st, t->ev_p, 0));
        const bool clip = cfg->grad_clip > 0.f && (!cfg->clip_first_step_only || *policy_steps_done == 0);
        if (clip) {
            CK(cudaMemsetAsync(t->sq, 0, sizeof(double), st));
            CKU(uhc_sqsum(pol.gfull, pol.nflat, t->sq, st), "gradient norm");
        }
        *adam_step_policy += 1; *policy_steps_done += 1;
        CKU(uhc_adam_step(pol.flat, pol.gfull, pol.adam_m, pol.adam_v, pol.nflat, pol.lr, 0.9f, 0.999f, 1e-8f, *adam_step_policy, clip ? t->sq : nullptr, clip ? cfg->grad_clip : 0.f, st), "policy Adam");
        for (const UhcNetDesc &n : t->pnets) if (refresh_bf16(n, st)) return -1;
    }
    return 0;
}

extern "C" {
static int trainer_create(const UhcNetDesc *pnets, int nprim, const UhcNetDesc *value, long max_rows, int max_envs, int device, UhcPpoTrainer **out) {
    const int npn = nprim > 0 ? nprim + 1 : 1;
    if (!pnets || !value || !out || max_rows <= 0 || max_envs <= 0 || nprim < 0 || nprim > 8) { uhc_err() = "uhc_ppo_trainer_create: bad argument"; return -2; }
    for (int j = 0; j < npn; j++) if (check_net(pnets[j], "policy")) return -2;
    if (check_net(*value, "value")) return -2;
    const int D = pnets[0].dims[0], A = pnets[0].dims[pnets[0].nlayers];
    if (D != value->dims[0] || value->dims[value->nlayers] != 1) { uhc_err() = "uhc_ppo_trainer_create: the nets must share the input width and the value head must be scalar"; return -2; }
    for (int j = 0; j < npn; j++) {
        const UhcNetDesc &n = pnets[j];
        if (n.dims[0] != D || n.flat != pnets[0].flat || n.gfull != pnets[0].gfull || n.nflat != pnets[0].nflat) { uhc_err() = "uhc_ppo_trainer_create: the policy's nets must share one flat parameter / gradient tensor and the observation"; return -2; }
        if (nprim > 0 && j < nprim && n.dims[n.nlayers] != A) { uhc_err() = "uhc_ppo_trainer_create: the primitives must share the action width"; return -2; }
        if (nprim > 0 && j == nprim && n.dims[n.nlayers] != nprim) { uhc_err() = "uhc_ppo_trainer_create: the composer's output width must be the number of primitives"; return -2; }
    }
    CK(cudaSetDevice(device));
    UhcPpoTrainer *t = new UhcPpoTrainer();
    t->device = device; t->cap = max_rows; t->cap_envs = max_envs; t->val = *value; t->nprim = nprim;
    t->pnets.assign(pnets, pnets + npn); t->pbufs.resize(npn);
    const long cap = max_rows, capp = pad64(max_rows);
    long maxN = 1, maxKh = 1;       // widest layer output; widest hidden input (layers i > 0)
    auto widths = [&](const UhcNetDesc &n) { for (int i = 0; i < n.nlayers; i++) { if (n.dims[i + 1] > maxN) maxN = n.dims[i + 1]; if (i > 0 && n.dims[i] > maxKh) maxKh = n.dims[i]; } };
    for (const UhcNetDesc &n : t->pnets) widths(n);
    widths(*value);
    int rc = 0;
    for (int j = 0; j < npn && !rc; j++) rc = alloc_net(t, t->pnets[j], t->pbufs[j], cap, !(nprim > 0 && j < nprim));
    rc = rc || alloc_net(t, t->val, t->vb, cap, true);
    if (nprim > 0) rc = rc || dalloc(t, &t->xall, (size_t)nprim * cap * A * 4, false) || dalloc(t, &t->dxall, (size_t)nprim * cap * A * 4, false) ||
                         dalloc(t, &t->mixw, (size_t)cap * nprim * 4, false) || dalloc(t, &t->dcomp, (size_t)cap * nprim * 4, false) || dalloc(t, &t->mean, (size_t)cap * A * 4, false);
    rc = rc || dalloc(t, &t->xb, (size_t)cap * pad64(D) * 2, true) || dalloc(t, &t->xT, (size_t)D * capp * 2, true) || dalloc(t, &t->lb, (size_t)max_envs * pad64(D) * 2, true);
    {   // scratch for the dW of layers with K % 4 != 0
        long need = 0;
        auto scan = [&](const UhcNetDesc &n) { for (int i = 0; i < n.nlayers; i++) if (n.dims[i] % 4) { const long v = (long)n.dims[i + 1] * ((n.dims[i] + 3) & ~3); if (v > need) need = v; } };
        for (auto &n : t->pnets) scan(n);
        scan(t->val);
        if (need) { void *p = nullptr; rc = rc || dalloc(t, &p, (size_t)need * 4, false); t->dWpad = (float *)p; t->dWpad_n = need; }
    }
    rc = rc || dalloc(t, &t->dz2, (size_t)cap * pad64(maxN) * 2, true) || dalloc(t, &t->dzT2, (size_t)maxN * capp * 2, true);
    rc = rc || dalloc(t, &t->dz, (size_t)cap * pad64(maxN) * 2, true) || dalloc(t, &t->dzT, (size_t)maxN * capp * 2, true) || dalloc(t, &t->hT, (size_t)maxKh * capp * 2, true) ||
         dalloc(t, &t->WT, (size_t)maxKh * pad64(maxN) * 2, true) || dalloc(t, &t->dh, (size_t)cap * maxKh * 4, false);
    rc = rc || dalloc(t, &t->dmean, (size_t)cap * A * 4, false) || dalloc(t, &t->dv, (size_t)cap * 4, false) || dalloc(t, &t->fixed, (size_t)cap * 4, false) ||
         dalloc(t, &t->adv, (size_t)cap * 4, false) || dalloc(t, &t->ret, (size_t)cap * 4, false) || dalloc(t, &t->last_v, (size_t)max_envs * 4, false) ||
         dalloc(t, &t->inv_count, 4, true) || dalloc(t, &t->mom, 16, true) || dalloc(t, &t->cnt, 8, true) || dalloc(t, &t->ntot, 8, true) || dalloc(t, &t->sq, 8, true);
    if (rc) { uhc_ppo_trainer_destroy(t); return -1; }
    CK(cudaStreamCreateWithFlags(&t->side, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&t->ev_ready, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&t->ev_v, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&t->ev_p, cudaEventDisableTiming));
    *out = t;
    return 0;
}
int uhc_ppo_trainer_create(const UhcNetDesc *policy, const UhcNetDesc *value, long max_rows, int max_envs, int device, UhcPpoTrainer **out) {
    return trainer_create(policy, 0, value, max_rows, max_envs, device, out);
}
int uhc_ppo_trainer_create_mcp(const UhcNetDesc *policy_nets, int nprim, const UhcNetDesc *value, long max_rows, int max_envs, int device, UhcPpoTrainer **out) {
    if (nprim < 1) { uhc_err() = "uhc_ppo_trainer_create_mcp: nprim >= 1"; return -2; }
    return trainer_create(policy_nets, nprim, value, max_rows, max_envs, device, out);
}

void uhc_ppo_trainer_destroy(UhcPpoTrainer *t) {
    if (!t) return;
    cudaSetDevice(t->device);
    for (void *p : t->allocs) cudaFree(p);
    for (auto &e : t->timing) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    if (t->ev_ready) cudaEventDestroy(t->ev_ready);
    if (t->ev_v) cudaEventDestroy(t->ev_v);
    if (t->ev_p) cudaEventDestroy(t->ev_p);
    if (t->side) cudaStreamDestroy(t->side);
    delete t;
}

int uhc_ppo_trainer_set_all_reduce(UhcPpoTrainer *t, UhcAllReduceFn fn) {
    if (!t) { uhc_err() = "uhc_ppo_trainer_set_all_reduce: null trainer"; return -2; }
    t->all_reduce = fn;
    return 0;
}

long uhc_ppo_kernel_launches(const UhcPpoTrainer *t) { return t ? t->launches : 0; }
const float *uhc_ppo_advantages(const UhcPpoTrainer *t) { return t ? t->adv : nullptr; }
const float *uhc_ppo_returns(const UhcPpoTrainer *t) { return t ? t->ret : nullptr; }

int uhc_ppo_comm_stats(UhcPpoTrainer *t, double *ms, long *bytes, int *calls) {
    if (!t) { uhc_err() = "uhc_ppo_comm_stats: null trainer"; return -2; }
    CK(cudaStreamSynchronize(t->side));
    double tot = 0.0;
    for (size_t i = 0; i < t->timing_used; i++) { float m = 0.f; CK(cudaEventElapsedTime(&m, t->timing[i].first, t->timing[i].second)); tot += m; }
    if (ms) *ms = tot;
    if (bytes) *bytes = t->comm_bytes;
    if (calls) *calls = t->comm_calls;
    t->timing_used = 0; t->comm_bytes = 0; t->comm_calls = 0;
    return 0;
}

int uhc_ppo_update_ex(UhcPpoTrainer *t, const float *states, const float *last_states, const float *actions, const float *rewards, const float *masks,
                      const float *exps, const float *log_std, int T, int E, const UhcPpoCfg *cfg, int *adam_step_policy, int *adam_step_value,
                      int *policy_steps_done, double *zfilter_stats, double *zfilter_sync, void *nccl_comm, int world, float *losses_out,
                      const float *extra_in, float *extra_out, long n_extra, void *stream) {
    if (!t || !states || !last_states || !actions || !rewards || !masks || !exps || !log_std || !cfg || !adam_step_policy || !adam_step_value || !policy_steps_done ||
        !losses_out || T <= 0 || E <= 0 || world < 1) { uhc_err() = "uhc_ppo_update: bad argument"; return -2; }
    if (n_extra < 0 || (n_extra > 0 && (!extra_in || !extra_out))) { uhc_err() = "uhc_ppo_update_ex: n_extra must be >= 0, with extra_in and extra_out when > 0"; return -2; }
    const long M = (long)T * E;
    if (M > t->cap || E > t->cap_envs) { uhc_err() = "uhc_ppo_update: the rollout exceeds the trainer's capacity"; return -2; }
    if (world > 1 && (!nccl_comm || !zfilter_stats || !zfilter_sync)) { uhc_err() = "uhc_ppo_update: world > 1 needs an ncclComm_t and the ZFilter statistics"; return -2; }
    CK(cudaSetDevice(t->device));
    cudaStream_t st = (cudaStream_t)stream;
    g_launches = 0;
    struct Tally { UhcPpoTrainer *t; ~Tally() { t->launches += g_launches; } } tally{t};
    const UhcNetDesc &pol = t->pnets[0], &val = t->val;      // pnets[0] carries the policy's flat parameter / gradient / Adam tensors
    const int D = pol.dims[0], A = pol.dims[pol.nlayers];
    const long Dp = pad64(D), Mp = pad64(M);
    void *comm = world > 1 ? nccl_comm : nullptr;
    const int nd = 4 + 1 + 2 * D;
    if (comm && (long)PLANES * nd > val.gtail) { uhc_err() = "uhc_ppo_update: the value net's gradient tail is too small for the statistics"; return -2; }
    if (comm && (long)PLANES * nd + n_extra > val.gtail) {
        uhc_err() = "uhc_ppo_update_ex: the value net's gradient tail holds " + std::to_string(val.gtail) + " floats, the statistics and the extra payload need " +
                    std::to_string((long)PLANES * nd + n_extra);
        return -2;
    }

    // ---- V(s_T) of the state after the last step, V(s) of every row (also epoch 0's value forward), GAE
    CKU(uhc_f32_to_bf16_padded(last_states, t->lb, E, D, (int)Dp, st), "bf16 last states");
    if (net_forward(val, t->vb, t->lb, E, false, st)) return -1;
    CK(cudaMemcpyAsync(t->last_v, t->vb.out, (size_t)E * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CKU(uhc_f32_to_bf16_padded(states, t->xb, (int)M, D, (int)Dp, st), "bf16 states");
    CKU(uhc_transpose_bf16(t->xb, t->xT, (int)M, D, (int)Dp, (int)Mp, st), "transpose states");
    if (net_forward(val, t->vb, t->xb, M, true, st)) return -1;
    CKU(uhc_gae(rewards, masks, t->vb.out, t->last_v, cfg->gamma, cfg->tau, t->adv, t->ret, T, E, st), "gae");
    CKU(uhc_adv_moments(t->adv, M, t->mom, st), "advantage moments");
    CK(cudaMemsetAsync(t->cnt, 0, sizeof(double), st));
    ++g_launches; k_count_selected<<<264, 256, 0, st>>>(exps, (size_t)M, t->cnt); CK(cudaGetLastError());
    float *tail = val.gfull + val.nflat;
    if (!comm) {
        CKU(uhc_adv_normalize(t->adv, M, t->mom, nullptr, st), "advantage normalisation");
        ++g_launches; k_inv_count<<<1, 1, 0, st>>>(t->cnt, t->inv_count); CK(cudaGetLastError());
    } else {
        CK(cudaMemsetAsync(tail, 0, (size_t)val.gtail * sizeof(float), st));
        ++g_launches; k_stats_pack<<<(nd + 255) / 256, 256, 0, st>>>(t->mom, (double)M, t->cnt, zfilter_stats, zfilter_sync, D, tail); CK(cudaGetLastError());
        if (n_extra) CK(cudaMemcpyAsync(tail + (size_t)PLANES * nd, extra_in, (size_t)n_extra * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if (!comm && n_extra) CK(cudaMemcpyAsync(extra_out, extra_in, (size_t)n_extra * sizeof(float), cudaMemcpyDeviceToDevice, st));   // one rank: the sum is the payload
    return run_epochs(t, actions, exps, log_std, M, cfg, adam_step_policy, adam_step_value, policy_steps_done, zfilter_stats, zfilter_sync, comm, world, comm != nullptr,
                      comm ? n_extra : 0, extra_out, true, losses_out, st);
}

int uhc_ppo_update(UhcPpoTrainer *t, const float *states, const float *last_states, const float *actions, const float *rewards, const float *masks,
                   const float *exps, const float *log_std, int T, int E, const UhcPpoCfg *cfg, int *adam_step_policy, int *adam_step_value,
                   int *policy_steps_done, double *zfilter_stats, double *zfilter_sync, void *nccl_comm, int world, float *losses_out, void *stream) {
    return uhc_ppo_update_ex(t, states, last_states, actions, rewards, masks, exps, log_std, T, E, cfg, adam_step_policy, adam_step_value, policy_steps_done,
                             zfilter_stats, zfilter_sync, nccl_comm, world, losses_out, nullptr, nullptr, 0, stream);
}

/* AgentPPO.update_policy (agent_ppo.py:16-51) alone: the epochs on caller-provided returns / (already normalised) advantages. */
int uhc_ppo_update_policy(UhcPpoTrainer *t, const float *states, const float *actions, const float *returns, const float *advantages, const float *exps,
                          const float *log_std, long M, const UhcPpoCfg *cfg, int *adam_step_policy, int *adam_step_value, int *policy_steps_done,
                          void *nccl_comm, int world, float *losses_out, void *stream) {
    if (!t || !states || !actions || !returns || !advantages || !exps || !log_std || !cfg || !adam_step_policy || !adam_step_value || !policy_steps_done || !losses_out ||
        M <= 0 || world < 1) { uhc_err() = "uhc_ppo_update_policy: bad argument"; return -2; }
    if (M > t->cap) { uhc_err() = "uhc_ppo_update_policy: the batch exceeds the trainer's capacity"; return -2; }
    // sharded, the policy gradient would be divided by this rank's selected-row count while the value gradient is divided by the global row
    // count; the global statistics travel only with uhc_ppo_update's collective
    if (world > 1) { uhc_err() = "uhc_ppo_update_policy: world > 1 is not supported (the global selected-row count is unknown here): use uhc_ppo_update"; return -2; }
    CK(cudaSetDevice(t->device));
    cudaStream_t st = (cudaStream_t)stream;
    g_launches = 0;
    struct Tally { UhcPpoTrainer *t; ~Tally() { t->launches += g_launches; } } tally{t};
    const int D = t->pnets[0].dims[0];
    CKU(uhc_f32_to_bf16_padded(states, t->xb, (int)M, D, (int)pad64(D), st), "bf16 states");
    CKU(uhc_transpose_bf16(t->xb, t->xT, (int)M, D, (int)pad64(D), (int)pad64(M), st), "transpose states");
    CK(cudaMemcpyAsync(t->adv, advantages, (size_t)M * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(t->ret, returns, (size_t)M * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemsetAsync(t->cnt, 0, sizeof(double), st));
    ++g_launches; k_count_selected<<<264, 256, 0, st>>>(exps, (size_t)M, t->cnt); CK(cudaGetLastError());
    ++g_launches; k_inv_count<<<1, 1, 0, st>>>(t->cnt, t->inv_count); CK(cudaGetLastError());
    return run_epochs(t, actions, exps, log_std, M, cfg, adam_step_policy, adam_step_value, policy_steps_done, nullptr, nullptr, nullptr, 1, false, 0, nullptr, false,
                      losses_out, st);
}
}  // extern "C"
