// eval.cu -- the device evaluation behind the C ABI (include/uhc_eval.h): deterministic roll-outs of whole clips, fail_safe and the
// per-frame imitation metrics, as CUDA-graph replays.
//
// Replaces one iteration of the chunk loop of AgentCopycat.eval_policy (uhc/agents/agent_copycat.py, kept as the default and as the
// reference of tests/test_gpu_eval.py).  One control step is
//   k_zfilter_apply_bf16, the policy GEMMs (+ mixture head), k_gauss_sample_dev   uhc_policy_forward's kernels, mean action, no ZFilter update
//   k_env_step                                                                   uhc_env_step under the engine's current (test-mode) cfg
//   k_eval_frame                                                                 per env still alive: the frame's metrics into a window buffer,
//                                                                                the reward sum, fail / end, the fail_safe flag
//   k_eval_export (SMPL export only)                                               per env that recorded a frame: its qpos as SMPL (export.cu)
//   k_eval_floor (floor rows only)                                                 per env that recorded a frame: its hulls against the floor (floor.cu)
//   k_eval_reseat (fail_safe only)                                               uhc_env_set_state_batch's re-seat of the flagged envs
// `window` steps are captured once per argument set into a CUDA graph (graph_cache.h); after each replay one 2-D copy moves the window's frame rows
// into the caller's (pinned) array and one 4-byte copy returns the number of envs still alive, the host loop's early exit.
//
// Compiled on its own with -fmad=false (uhc_b200/build.py) like motion_lib.cu: k_eval_frame restates numpy's fp64 arithmetic
// (eval_core.h) without contracted multiply-adds.  The policy and physics kernels it replays are compiled with the rest of the library.
#include <cuda_runtime.h>
#include <limits.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_eval.h"
#include "errors.h"
#include "eval_core.h"
#include "eval_glue.h"
#include "floor_core.h"
#include "graph_cache.h"
#include "sim_core.h"
#include "smpl_export_core.h"
#include "track_glue.h"

using namespace uhc;

namespace {

constexpr int NCOL = evalm::EV_N, NSTATE = UHC_EVAL_STATE, RING = 2 * 144;   // ring per env: pred xpos72 + gt wbpos72 of the two previous frames
static_assert(NCOL == UHC_EVAL_NCOL, "eval_core.h and uhc_eval.h disagree on the frame columns");

// one thread per env i < n: the recorded frame of this step (host loop: get_states of the live envs, traj append, rsum += r,
// fail -> set_states or alive = False, end -> alive = False)
template <class Real>
__global__ void __launch_bounds__(128) k_eval_frame(const Real *__restrict__ state, const int *__restrict__ istate, const Real *__restrict__ expert,
                                                    const int *__restrict__ clip_adr, const float *__restrict__ rew, const int *__restrict__ fail,
                                                    const int *__restrict__ end, int n, int nrec_max, int fail_safe, int window, int slot,
                                                    UhcEvalClip *__restrict__ clips, int *__restrict__ alive, int *__restrict__ reseat,
                                                    double *__restrict__ ring, double *__restrict__ win, double *__restrict__ win_states,
                                                    int *__restrict__ alive_count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    reseat[i] = 0;
    if (alive[i]) {
        UhcEvalClip c = clips[i];
        const int k = c.frames;
        if (k >= nrec_max) alive[i] = 0;       // the host loop's step limit, max(len) - 1: only the tail of the last window steps past it
        else {
            const int *is = istate + (size_t)i * SI_SIZE;
            const int cur_t = is[SI_CUR_T], clip = is[SI_CLIP];
            const int a0 = clip_adr[clip], len = clip_adr[clip + 1] - a0;
            const Real *gt = expert + ((size_t)a0 + (cur_t < len - 1 ? cur_t : len - 1)) * EX_SIZE;
            const Real *st = state + (size_t)i * ST_SIZE;
            double pq[7], gq[7], pj[72], gj[72];
            for (int j = 0; j < 7; j++) { pq[j] = (double)st[ST_Q + j]; gq[j] = (double)gt[EX_QPOS + j]; }
            for (int j = 0; j < 72; j++) { pj[j] = (double)st[ST_XPOS + j]; gj[j] = (double)gt[EX_WBPOS + j]; }
            double *r = ring + (size_t)i * RING;
            double *cur = r + (k & 1) * 144, *prev = r + ((k + 1) & 1) * 144;     // prev: frame k - 1; cur (before it is overwritten): frame k - 2
            double out[NCOL];
            evalm::eval_frame(pq, gq, pj, gj, k >= 1 ? prev : nullptr, k >= 1 ? prev + 72 : nullptr, k >= 2 ? cur : nullptr, k >= 2 ? cur + 72 : nullptr, out);
            for (int j = 0; j < 72; j++) { cur[j] = pj[j]; cur[72 + j] = gj[j]; }
            double *w = win + ((size_t)i * window + slot) * NCOL;
            for (int j = 0; j < NCOL; j++) w[j] = out[j];
            if (win_states) {
                double *ws = win_states + ((size_t)i * window + slot) * NSTATE;
                for (int j = 0; j < 76; j++) ws[j] = (double)st[ST_Q + j];
                for (int j = 0; j < 72; j++) ws[76 + j] = pj[j];
            }
            c.frames = k + 1; c.last_t = cur_t; c.reward_sum += (double)rew[i];
            const bool f = fail[i] != 0, d = end[i] != 0;
            if (f) { c.fail_any = 1; if (fail_safe) reseat[i] = 1; else alive[i] = 0; }
            if (d) alive[i] = 0;
            clips[i] = c;
        }
    }
    if (alive_count && alive[i]) atomicAdd(alive_count, 1);
}

__global__ void k_eval_init(int n, UhcEvalClip *__restrict__ clips, int *__restrict__ alive, int *__restrict__ reseat, unsigned char *__restrict__ ones, int E) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { UhcEvalClip c; c.frames = 0; c.last_t = 0; c.fail_any = 0; c.reserved = 0; c.reward_sum = 0.0; clips[i] = c; alive[i] = 1; reseat[i] = 0; }
    if (i < E) ones[i] = 1;
}

// the policies of one call: group g on env rows [row0[g], row0[g + 1]).  A single-policy call is one group over rows 0 .. n-1 that takes
// the ungrouped kernels and the caller's log_std
struct EvalPolicies { bool grouped; std::vector<evalx::Policy> pols; std::vector<int> row0; const float *log_std; const double *const *zstats; };

struct EvalCtx {
    UhcEngine *eng = nullptr;
    int E = 0, n_cap = 0, win_cap = 0, states_cap = 0;
    size_t smpl_cap = 0, floor_cap = 0;           // rows (env x slot) of d_wsmpl, d_wfloor
    unsigned long long gen = 0;                   // bumped when the scratch below is reallocated
    UhcEvalClip *d_clips = nullptr; int *d_alive = nullptr, *d_reseat = nullptr, *d_count = nullptr; unsigned char *d_ones = nullptr;
    double *d_ring = nullptr, *d_win = nullptr, *d_wstates = nullptr;
    double *d_wsmpl = nullptr; int *d_xdone = nullptr;   // SMPL export: window rows [n][window][UHC_EVAL_SMPL], frames exported per env
    double *d_wfloor = nullptr, *d_fprev = nullptr; int *d_fdone = nullptr;   // floor rows: window rows [n][window][NCOL], per env the qpos last measured, frames measured
    int *h_count = nullptr;                       // pinned
    cudaEvent_t ev = nullptr;
    std::vector<int> ids, clip0, start, len;      // reset arguments (kept: no allocation in the steady state)
    GraphCache graphs{32}, ggraphs{16};           // of uhc_eval_run and of uhc_eval_run_groups (graph_cache.h)
};
std::vector<EvalCtx *> g_ev;

EvalCtx *ev_ctx(UhcEngine *e) {
    for (EvalCtx *c : g_ev) if (c->eng == e) return c;
    EvalCtx *c = new EvalCtx(); c->eng = e; c->E = uhc_num_envs(e);
    g_ev.push_back(c);
    return c;
}
// per-env arrays sized by E once; the window buffers grow with n * window (and the state record and the SMPL export with it when requested).
// Called before any capture: a graph holds these pointers, so they never change while one of them can be replayed (gen)
int ensure(EvalCtx *c, int n, int window, bool states, bool smpl, bool floor) {
    const size_t E = c->E;
    if (!c->d_clips) {
        CK(cudaMalloc((void **)&c->d_clips, E * sizeof(UhcEvalClip))); CK(cudaMalloc((void **)&c->d_alive, E * 4)); CK(cudaMalloc((void **)&c->d_reseat, E * 4));
        CK(cudaMalloc((void **)&c->d_count, 4)); CK(cudaMalloc((void **)&c->d_ones, E)); CK(cudaMalloc((void **)&c->d_ring, E * RING * sizeof(double)));
        CK(cudaHostAlloc((void **)&c->h_count, 4, cudaHostAllocDefault)); CK(cudaEventCreateWithFlags(&c->ev, cudaEventDisableTiming));
        c->gen++;
    }
    const int need = n * window;
    if (need > c->win_cap) {
        if (c->d_win) cudaFree(c->d_win);
        CK(cudaMalloc((void **)&c->d_win, (size_t)need * NCOL * sizeof(double))); c->win_cap = need; c->gen++;
    }
    if (states && need > c->states_cap) {
        if (c->d_wstates) cudaFree(c->d_wstates);
        CK(cudaMalloc((void **)&c->d_wstates, (size_t)need * NSTATE * sizeof(double))); c->states_cap = need; c->gen++;
    }
    if (smpl && (size_t)need > c->smpl_cap) {
        if (c->d_wsmpl) cudaFree(c->d_wsmpl);
        c->d_wsmpl = nullptr; c->smpl_cap = 0; c->gen++;
        CK(cudaMalloc((void **)&c->d_wsmpl, (size_t)need * UHC_EVAL_SMPL * sizeof(double))); c->smpl_cap = (size_t)need;
    }
    if (smpl && !c->d_xdone) { CK(cudaMalloc((void **)&c->d_xdone, E * sizeof(int))); c->gen++; }
    if (floor && (size_t)need > c->floor_cap) {
        if (c->d_wfloor) cudaFree(c->d_wfloor);
        c->d_wfloor = nullptr; c->floor_cap = 0; c->gen++;
        CK(cudaMalloc((void **)&c->d_wfloor, (size_t)need * floorm::NCOL * sizeof(double))); c->floor_cap = (size_t)need;
    }
    if (floor && !c->d_fdone) {
        CK(cudaMalloc((void **)&c->d_fdone, E * sizeof(int))); CK(cudaMalloc((void **)&c->d_fprev, E * motion::MQ * sizeof(double))); c->gen++;
    }
    return 0;
}

int enqueue_window(EvalCtx *c, const evalx::EngineRefs &R, const EvalPolicies &P, float zclip, int n, int nrec_max, int fail_safe, int window, bool states,
                   bool smpl, bool floor, cudaStream_t st) {
    for (int s = 0; s < window; s++) {
        const int rc = P.grouped ? evalx::groups_enqueue(c->eng, P.pols, P.row0.data(), P.zstats, zclip, R.obs, c->d_ones, R.act, st)
                                 : evalx::policy_enqueue(c->eng, P.pols[0], R.obs, P.log_std, (double *)P.zstats[0], zclip, c->d_ones, R.act, st);
        if (rc) return rc;
        if (uhc_env_step(c->eng, R.act, R.obs, R.rew, R.cinfo, R.fail, R.end, R.pct, nullptr, st)) return uhc_err_prefix("env step");
        const bool last = s == window - 1;
        if (last) CK(cudaMemsetAsync(c->d_count, 0, 4, st));
        if (R.precision == 32)
            k_eval_frame<float><<<(n + 127) / 128, 128, 0, st>>>((const float *)R.state, R.istate, (const float *)R.expert, R.clip_adr, R.rew, R.fail, R.end, n, nrec_max,
                                                                fail_safe, window, s, c->d_clips, c->d_alive, c->d_reseat, c->d_ring, c->d_win,
                                                                states ? c->d_wstates : nullptr, last ? c->d_count : nullptr);
        else
            k_eval_frame<double><<<(n + 127) / 128, 128, 0, st>>>((const double *)R.state, R.istate, (const double *)R.expert, R.clip_adr, R.rew, R.fail, R.end, n, nrec_max,
                                                                 fail_safe, window, s, c->d_clips, c->d_alive, c->d_reseat, c->d_ring, c->d_win,
                                                                 states ? c->d_wstates : nullptr, last ? c->d_count : nullptr);
        CK(cudaGetLastError());
        if (smpl) CK(smplx::launch_eval_export(R.precision, R.state, R.istate, trackx::clip_models(c->eng), trackx::motion_model(c->eng).body, c->d_clips,
                                                c->d_xdone, n, window, s, c->d_wsmpl, st));
        if (floor) CK(floorm::launch_eval_floor(c->eng, R.precision, R.state, R.istate, trackx::clip_models(c->eng), c->d_clips, c->d_fdone, c->d_fprev, n,
                                                window, s, c->d_wfloor, st));
        if (fail_safe) CK(evalx::launch_reseat(c->eng, n, c->d_reseat, st));
    }
    return 0;
}

// reset: idle envs parked on the chunk's first clip, then envs 0..n-1 on their clips from frame 0 (the host loop's order)
int reset_envs(EvalCtx *c, UhcEngine *e, const evalx::EngineRefs &R, int n, const int *clip_host, cudaStream_t st) {
    if (n < R.E) {
        const int m = R.E - n;
        c->ids.resize(m); c->clip0.assign(m, clip_host[0]); c->start.assign(m, 0); c->len.assign(m, R.clip_len_h[clip_host[0]]);
        for (int k = 0; k < m; k++) c->ids[k] = n + k;
        if (uhc_env_reset(e, m, c->ids.data(), c->clip0.data(), c->start.data(), c->len.data(), nullptr, nullptr, R.obs, st)) return uhc_err_prefix("reset");
    }
    c->ids.resize(n); c->start.assign(n, 0); c->len.resize(n);
    for (int k = 0; k < n; k++) { c->ids[k] = k; c->len[k] = R.clip_len_h[clip_host[k]]; }
    if (uhc_env_reset(e, n, c->ids.data(), clip_host, c->start.data(), c->len.data(), nullptr, nullptr, R.obs, st)) return uhc_err_prefix("reset");
    k_eval_init<<<(R.E + 127) / 128, 128, 0, st>>>(n, c->d_clips, c->d_alive, c->d_reseat, c->d_ones, R.E);
    CK(cudaGetLastError());
    return 0;
}

// replays until every env has stopped or nrec_max steps have run; after each, the window's rows of envs 0..n-1 go to the caller's arrays
int replay(EvalCtx *c, cudaGraphExec_t exec, int n, int nrec_max, int window, const UhcEvalOut &o, cudaStream_t st) {
    double *frames_host = o.frames_host, *states_host = o.states_host_or_null, *smpl_host = o.smpl_host_or_null, *floor_host = o.floor_host_or_null;
    if (smpl_host && (!c->d_wsmpl || c->smpl_cap < (size_t)n * (size_t)window)) { uhc_err() = "SMPL export: the window buffer is smaller than n * window rows"; return -1; }
    for (int s0 = 0; s0 < nrec_max; s0 += window) {
        CK(cudaGraphLaunch(exec, st));
        const int rows = nrec_max - s0 < window ? nrec_max - s0 : window;
        CK(cudaMemcpy2DAsync(frames_host + (size_t)s0 * NCOL, (size_t)nrec_max * NCOL * sizeof(double), c->d_win, (size_t)window * NCOL * sizeof(double),
                              (size_t)rows * NCOL * sizeof(double), n, cudaMemcpyDeviceToHost, st));
        if (states_host)
            CK(cudaMemcpy2DAsync(states_host + (size_t)s0 * NSTATE, (size_t)nrec_max * NSTATE * sizeof(double), c->d_wstates, (size_t)window * NSTATE * sizeof(double),
                                  (size_t)rows * NSTATE * sizeof(double), n, cudaMemcpyDeviceToHost, st));
        if (smpl_host)
            CK(cudaMemcpy2DAsync(smpl_host + (size_t)s0 * UHC_EVAL_SMPL, (size_t)nrec_max * UHC_EVAL_SMPL * sizeof(double), c->d_wsmpl,
                                  (size_t)window * UHC_EVAL_SMPL * sizeof(double), (size_t)rows * UHC_EVAL_SMPL * sizeof(double), n, cudaMemcpyDeviceToHost, st));
        if (floor_host)
            CK(cudaMemcpy2DAsync(floor_host + (size_t)s0 * floorm::NCOL, (size_t)nrec_max * floorm::NCOL * sizeof(double), c->d_wfloor,
                                  (size_t)window * floorm::NCOL * sizeof(double), (size_t)rows * floorm::NCOL * sizeof(double), n, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(c->h_count, c->d_count, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(c->ev, st));
        CK(cudaEventSynchronize(c->ev));
        if (*c->h_count == 0) break;
    }
    CK(cudaMemcpyAsync(o.clips_host, c->d_clips, (size_t)n * sizeof(UhcEvalClip), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
}

// One chunk: G policies side by side, group g on envs [row0[g], row0[g] + group_n[g]); uhc_eval_run is the ungrouped call of one group
int eval_run(UhcEngine *e, bool grouped, int G, const int *group_n, const int *clip_host, const UhcMlp *mlps, const UhcMcp *mcps, const float *log_std,
             const double *const *zstats, float zclip, int fail_safe, int window, const UhcEvalOut &o, void *stream) {
    const std::string who = std::string(grouped ? "uhc_eval_run_groups" : "uhc_eval_run") + (mcps ? "_mcp" : "");
    auto refuse = [&](const char *why) { uhc_err() = who + ": " + why; return -2; };
    if (!e || !group_n || !clip_host || (!mlps && !mcps) || !zstats || (!grouped && (!log_std || !zstats[0])) || !o.frames_host || !o.clips_host) return refuse("null argument");
    if (G < 1 || G > UHC_EVAL_MAX_GROUPS) return refuse("G must be 1 .. UHC_EVAL_MAX_GROUPS");
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    if (!grouped && (group_n[0] < 1 || group_n[0] > R.E)) return refuse("n must be 1 .. E");
    EvalPolicies P{grouped, std::vector<evalx::Policy>(G), std::vector<int>(G + 1, 0), log_std, zstats};
    for (int g = 0; g < G; g++) {
        if (group_n[g] < 1) return refuse("every group needs at least one env");
        if (!zstats[g]) return refuse("null ZFilter statistics");
        P.row0[g + 1] = P.row0[g] + group_n[g];
        if (P.row0[g + 1] > R.E) return refuse("the groups hold more than E envs");
    }
    const int n = P.row0[G];
    if (window < 1) return refuse("window < 1");
    if ((long long)n * window > INT_MAX) return refuse("n * window exceeds INT_MAX window rows");
    if (R.num_clips <= 0) return refuse("no clips loaded");
    int max_len = 0;
    for (int i = 0; i < n; i++) {
        if (clip_host[i] < 0 || clip_host[i] >= R.num_clips) return refuse("clip index out of range");
        max_len = R.clip_len_h[clip_host[i]] > max_len ? R.clip_len_h[clip_host[i]] : max_len;
    }
    unsigned long long pgen = 0;
    int rc = grouped ? evalx::groups_prepare(e, G, mlps, mcps, &P.pols, &pgen) : evalx::policy_prepare(e, mlps, mcps, &P.pols[0], &pgen);
    if (rc) return rc;
    EvalCtx *c = ev_ctx(e);
    const bool states = o.states_host_or_null != nullptr, smpl = o.smpl_host_or_null != nullptr, floor = o.floor_host_or_null != nullptr;
    const unsigned long long fgen = floor ? floorm::floor_gen(e) : 0;
    if (floor && !fgen) return refuse("floor rows need the hull vertices (uhc_floor_init)");
    if (ensure(c, n, window, states, smpl, floor)) return -1;
    cudaStream_t st = (cudaStream_t)stream;
    const int nrec_max = max_len - 1;
    if (reset_envs(c, e, R, n, clip_host, st)) return -1;
    if (smpl) CK(cudaMemsetAsync(c->d_xdone, 0, (size_t)n * sizeof(int), st));
    if (floor) CK(cudaMemsetAsync(c->d_fdone, 0, (size_t)n * sizeof(int), st));
    // no grouped policy covers the parked envs: they step with zero actions (the graph writes action rows 0 .. n-1 only)
    if (grouped && n < R.E) CK(cudaMemsetAsync(R.act + (size_t)n * R.act_dim, 0, (size_t)(R.E - n) * R.act_dim * sizeof(float), st));

    // the key: every argument the graph's kernels got.  The generations: the graph also holds the policy scratch, the window buffers and
    // the engine view (cfg, clip table) of its capture, and is dropped once any of them has changed
    struct { int n, nrec_max, window, fail_safe, states, smpl; float zclip; unsigned long long floor; const float *log_std; } head;
    memset(&head, 0, sizeof head);
    head.n = n; head.nrec_max = nrec_max; head.window = window; head.fail_safe = fail_safe ? 1 : 0; head.states = states; head.smpl = smpl; head.floor = fgen; head.zclip = zclip;
    head.log_std = log_std;
    std::string key;
    GraphCache::append(&key, &head); GraphCache::append(&key, group_n, G); GraphCache::append(&key, zstats, G); GraphCache::append(&key, P.pols.data(), G);
    const GraphCache::Gens gens{pgen, c->gen, R.view_gen};
    GraphCache &cache = grouped ? c->ggraphs : c->graphs;
    cache.drop_stale(gens);
    cudaGraphExec_t exec = cache.find(key);
    if (!exec) {
        rc = GraphCache::capture([&](cudaStream_t cs) { return enqueue_window(c, R, P, zclip, n, nrec_max, head.fail_safe, window, states, smpl, floor, cs); }, &exec);
        if (rc) return rc;
        cache.insert(std::move(key), gens, exec);
    }
    return replay(c, exec, n, nrec_max, window, o, st);
}

}  // namespace

extern "C" {

static UhcEvalOut eval_out(double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null) {
    UhcEvalOut o; o.frames_host = frames_host; o.clips_host = clips_host; o.states_host_or_null = states_host_or_null; o.smpl_host_or_null = nullptr; o.floor_host_or_null = nullptr;
    return o;
}

int uhc_eval_run(UhcEngine *e, int n, const int *clip_host, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats, float zclip,
                 int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream) {
    const UhcEvalOut o = eval_out(frames_host, clips_host, states_host_or_null);
    return uhc_eval_run_ex(e, n, clip_host, mlp, log_std, zfilter_stats, zclip, fail_safe, window, &o, stream);
}
int uhc_eval_run_mcp(UhcEngine *e, int n, const int *clip_host, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats, float zclip,
                     int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream) {
    const UhcEvalOut o = eval_out(frames_host, clips_host, states_host_or_null);
    return uhc_eval_run_mcp_ex(e, n, clip_host, mcp, log_std, zfilter_stats, zclip, fail_safe, window, &o, stream);
}

int uhc_eval_run_groups(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMlp *mlps, const double *const *zfilter_stats_host,
                        float zclip, int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream) {
    const UhcEvalOut o = eval_out(frames_host, clips_host, states_host_or_null);
    return uhc_eval_run_groups_ex(e, G, group_n_host, clip_host, mlps, zfilter_stats_host, zclip, fail_safe, window, &o, stream);
}
int uhc_eval_run_groups_mcp(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMcp *mcps, const double *const *zfilter_stats_host,
                            float zclip, int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream) {
    const UhcEvalOut o = eval_out(frames_host, clips_host, states_host_or_null);
    return uhc_eval_run_groups_mcp_ex(e, G, group_n_host, clip_host, mcps, zfilter_stats_host, zclip, fail_safe, window, &o, stream);
}

int uhc_eval_run_ex(UhcEngine *e, int n, const int *clip_host, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats, float zclip,
                    int fail_safe, int window, const UhcEvalOut *out, void *stream) {
    if (!mlp) { uhc_err() = "uhc_eval_run: null policy"; return -2; }
    if (!out) { uhc_err() = "uhc_eval_run: null output struct"; return -2; }
    return eval_run(e, false, 1, &n, clip_host, mlp, nullptr, log_std, &zfilter_stats, zclip, fail_safe, window, *out, stream);
}
int uhc_eval_run_mcp_ex(UhcEngine *e, int n, const int *clip_host, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats, float zclip,
                        int fail_safe, int window, const UhcEvalOut *out, void *stream) {
    if (!mcp) { uhc_err() = "uhc_eval_run_mcp: null policy"; return -2; }
    if (!out) { uhc_err() = "uhc_eval_run_mcp: null output struct"; return -2; }
    return eval_run(e, false, 1, &n, clip_host, nullptr, mcp, log_std, &zfilter_stats, zclip, fail_safe, window, *out, stream);
}
int uhc_eval_run_groups_ex(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMlp *mlps, const double *const *zfilter_stats_host,
                           float zclip, int fail_safe, int window, const UhcEvalOut *out, void *stream) {
    if (!mlps) { uhc_err() = "uhc_eval_run_groups: null policy"; return -2; }
    if (!out) { uhc_err() = "uhc_eval_run_groups: null output struct"; return -2; }
    return eval_run(e, true, G, group_n_host, clip_host, mlps, nullptr, nullptr, zfilter_stats_host, zclip, fail_safe, window, *out, stream);
}
int uhc_eval_run_groups_mcp_ex(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMcp *mcps, const double *const *zfilter_stats_host,
                               float zclip, int fail_safe, int window, const UhcEvalOut *out, void *stream) {
    if (!mcps) { uhc_err() = "uhc_eval_run_groups_mcp: null policy"; return -2; }
    if (!out) { uhc_err() = "uhc_eval_run_groups_mcp: null output struct"; return -2; }
    return eval_run(e, true, G, group_n_host, clip_host, nullptr, mcps, nullptr, zfilter_stats_host, zclip, fail_safe, window, *out, stream);
}

int uhc_eval_graph_count(const UhcEngine *e) {
    for (const EvalCtx *c : g_ev) if (c->eng == e) return (int)(c->graphs.size() + c->ggraphs.size());
    return 0;
}

void uhc_eval_release(UhcEngine *e) {
    for (size_t i = 0; i < g_ev.size(); i++) if (g_ev[i]->eng == e) {
        EvalCtx *c = g_ev[i];
        c->graphs.clear(); c->ggraphs.clear();
        for (void *p : {(void *)c->d_clips, (void *)c->d_alive, (void *)c->d_reseat, (void *)c->d_count, (void *)c->d_ones, (void *)c->d_ring,
                        (void *)c->d_win, (void *)c->d_wstates, (void *)c->d_wsmpl, (void *)c->d_xdone, (void *)c->d_wfloor, (void *)c->d_fprev, (void *)c->d_fdone}) if (p) cudaFree(p);
        if (c->h_count) cudaFreeHost(c->h_count);
        if (c->ev) cudaEventDestroy(c->ev);
        delete c; g_ev.erase(g_ev.begin() + i); return;
    }
}

}  // extern "C"
