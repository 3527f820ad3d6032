// track.cu -- the batched physics tracker behind the C ABI (include/uhc_track.h): target frames streamed one per control step into a
// per-env window of expert-table rows, and one CUDA-graph replay per step of
//   k_track_push  (when frames are passed)   per env: rebase a full window, the record of the new frame (track_core.h)
//   k_track_gate                             per env: an env whose row cur_t + 1 was never pushed gets an invalid record for this step
//   k_track_obs   (step_kernel.cu)           the observation of the stored state against row cur_t + 1 (track_obs.h)
//   ZFilter + policy GEMMs + mean action     uhc_eval_run's kernels (rollout.cu)
//   k_env_step                               unchanged, obs = null
//   k_track_post                             per env: the gated record restored, step count, fail_safe flag, the state gathered
//   k_eval_reseat (fail_safe only)           uhc_eval_run's re-seat on row cur_t
//
// Compiled on its own with -fmad=false (uhc_b200/build.py) like motion_lib.cu: the rows restate motion_lib.py's fp64 arithmetic and
// must equal uhc_load_motions' rows bit for bit.
#include <cuda_runtime.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_track.h"
#include "eval_glue.h"
#include "track_glue.h"
#include "track_core.h"
#include "sim_core.h"

using namespace uhc;

static thread_local std::string g_tr_err;
#define CKT(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { g_tr_err = std::string(#x) + ": " + cudaGetErrorString(e_); return -1; } } while (0)

namespace {

using motion::MotionModel;
using motion::REC;

// reset: frames [n][2][row_w] -> rows 0, 1 of env ids[i]
template <class Out>
__global__ void k_track_rows(MotionModel m, int kind, int pose_dim, int row_w, int H, int n, const int *__restrict__ ids, const double *__restrict__ frames,
                             const int *__restrict__ fk, Out *__restrict__ table, double *__restrict__ raw, int *__restrict__ have,
                             int *__restrict__ steps, int *__restrict__ dropped) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int env = ids[i];
    int h = 0;
    motion::track_reset_rows<Out>(m, kind, pose_dim, row_w, fk ? fk[env] : 0, frames + (size_t)i * 2 * row_w, table + (size_t)env * H * REC,
                                  raw + (size_t)env * 2 * row_w, &h);
    have[env] = h; steps[env] = 0; dropped[env] = 0;
}

// push: frame next[env] onto every masked-in env that was reset onto its stream
template <class Out>
__global__ void k_track_push(MotionModel m, int kind, int pose_dim, int row_w, int H, int E, const double *__restrict__ next, const int *__restrict__ mask,
                             const int *__restrict__ fk, Out *__restrict__ table, int *__restrict__ istate, double *__restrict__ raw,
                             int *__restrict__ have, int *__restrict__ dropped) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= E || (mask && !mask[env])) return;
    int *is = istate + (size_t)env * SI_SIZE;
    if (is[SI_LEN] != H || is[SI_CLIP] != env) return;      // not reset onto its stream since the table was installed
    int h = have[env], ct = is[SI_CUR_T];
    if (motion::track_push_row<Out>(m, kind, pose_dim, row_w, fk ? fk[env] : 0, H, next + (size_t)env * row_w, table + (size_t)env * H * REC,
                                    raw + (size_t)env * 2 * row_w, &h, &ct)) { have[env] = h; is[SI_CUR_T] = ct; }
    else dropped[env]++;
}

// status[env]: 0 = stepped on its stream, > 0 = a valid record the step kernel must skip (no row cur_t + 1, or not a stream record):
// its length + 1, restored by k_track_post; -1 = an invalid record the step kernel skips by itself
__global__ void k_track_gate(int *__restrict__ istate, const int *__restrict__ have, int H, int E, int num_clips, int *__restrict__ status) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= E) return;
    int *is = istate + (size_t)env * SI_SIZE;
    const int len = is[SI_LEN], clip = is[SI_CLIP];
    if (!(len >= 2 && clip >= 0 && clip < num_clips)) { status[env] = -1; return; }
    if (clip == env && len == H && is[SI_CUR_T] + 1 < have[env]) { status[env] = 0; return; }
    status[env] = len + 1;
    is[SI_LEN] = 0;
}

__global__ void k_track_ungate(int *__restrict__ istate, const int *__restrict__ status, int E) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env < E && status[env] > 0) istate[(size_t)env * SI_SIZE + SI_LEN] = status[env] - 1;
}

// one warp per env: the gated record restored, the step count, the fail_safe flag, state_out = qpos 76 | qvel 75 | xpos 72
template <class Real>
__global__ void __launch_bounds__(128) k_track_post(const Real *__restrict__ state, int *__restrict__ istate, const int *__restrict__ status,
                                                    const int *__restrict__ fail, int fail_safe, int E, int *__restrict__ steps, int *__restrict__ reseat,
                                                    Real *__restrict__ out) {
    const int env = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (env >= E) return;
    const int s = status[env];
    if (lane == 0) {
        if (s > 0) istate[(size_t)env * SI_SIZE + SI_LEN] = s - 1;
        if (s == 0) steps[env]++;
        reseat[env] = fail_safe && s == 0 && fail[env] != 0;
    }
    const Real *st = state + (size_t)env * ST_SIZE;
    Real *o = out + (size_t)env * UHC_TRACK_OUT;
    for (int k = lane; k < NQ; k += 32) o[k] = st[ST_Q + k];
    for (int k = lane; k < NV; k += 32) o[NQ + k] = st[ST_V + k];
    for (int k = lane; k < 72; k += 32) o[NQ + NV + k] = st[ST_XPOS + k];
}

__global__ void k_fill_ones(unsigned char *p, int n) { const int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = 1; }

struct TrackKey {
    int has_next, has_mask, fail_safe, nprim; float zclip; unsigned long long scratch_gen, track_gen, view_gen;
    UhcMlp nets[UHC_MCP_MAX_PRIM + 1]; const float *log_std; const double *zstats; void *out; float *rew; int *fail;
    bool operator==(const TrackKey &o) const { return memcmp(this, &o, sizeof(TrackKey)) == 0; }
};
struct TrackCtx {
    UhcEngine *eng = nullptr;
    int E = 0, H = 0, kind = 0, pose_dim = 0, row_w = 0;
    unsigned long long table_gen = 0, gen = 0;
    double *d_raw = nullptr, *d_next = nullptr;
    int *d_have = nullptr, *d_steps = nullptr, *d_dropped = nullptr, *d_status = nullptr, *d_reseat = nullptr, *d_mask = nullptr, *d_fk = nullptr, *d_ids = nullptr;
    unsigned char *d_ones = nullptr;
    int *h_ids = nullptr;                          // pinned staging of the reset's env ids
    cudaEvent_t ids_done = nullptr;                // the last k_track_rows that read d_ids has been enqueued before it
    std::vector<int> zeros, lens;                  // reset arguments of uhc_env_reset (start 0, length H)
    std::vector<std::pair<TrackKey, cudaGraphExec_t>> graphs;
};
std::vector<TrackCtx *> g_tr;
unsigned long long g_tr_gen = 0;                   // distinct per begin: graphs never outlive the buffers they hold

TrackCtx *find_ctx(UhcEngine *e) { for (TrackCtx *c : g_tr) if (c->eng == e) return c; return nullptr; }
void free_ctx(TrackCtx *c) {
    cudaDeviceSynchronize();
    for (auto &g : c->graphs) cudaGraphExecDestroy(g.second);
    for (void *p : {(void *)c->d_raw, (void *)c->d_next, (void *)c->d_have, (void *)c->d_steps, (void *)c->d_dropped, (void *)c->d_status, (void *)c->d_reseat,
                    (void *)c->d_mask, (void *)c->d_fk, (void *)c->d_ids, (void *)c->d_ones}) if (p) cudaFree(p);
    if (c->h_ids) cudaFreeHost(c->h_ids);
    if (c->ids_done) cudaEventDestroy(c->ids_done);
    for (size_t i = 0; i < g_tr.size(); i++) if (g_tr[i] == c) { g_tr.erase(g_tr.begin() + i); break; }
    delete c;
}

// the tracker of e while its table is still the engine's table and its cfg can run the stream, else null with the reason in g_tr_err
TrackCtx *live_ctx(UhcEngine *e, const char *who) {
    TrackCtx *c = e ? find_ctx(e) : nullptr;
    if (!c) { g_tr_err = std::string(who) + ": not tracking (uhc_track_begin)"; return nullptr; }
    if (trackx::table_gen(e) != c->table_gen) { g_tr_err = std::string(who) + ": tracking ended: the clip table was replaced"; return nullptr; }
    if (const char *why = trackx::cfg_error(e, c->H)) { g_tr_err = std::string(who) + ": " + why; return nullptr; }
    return c;
}

int enqueue_push(TrackCtx *c, const evalx::EngineRefs &R, const double *next, const int *mask, cudaStream_t st) {
    const int E = c->E, nb = (E + 127) / 128;
    const MotionModel &m = trackx::motion_model(c->eng);
    if (R.precision == 32)
        k_track_push<float><<<nb, 128, 0, st>>>(m, c->kind, c->pose_dim, c->row_w, c->H, E, next, mask, c->d_fk, (float *)R.expert, R.istate, c->d_raw,
                                                c->d_have, c->d_dropped);
    else
        k_track_push<double><<<nb, 128, 0, st>>>(m, c->kind, c->pose_dim, c->row_w, c->H, E, next, mask, c->d_fk, (double *)R.expert, R.istate, c->d_raw,
                                                 c->d_have, c->d_dropped);
    CKT(cudaGetLastError());
    return 0;
}

int enqueue_step(TrackCtx *c, const evalx::EngineRefs &R, const TrackKey &k, const UhcMlp *mlp, const UhcMcp *mcp, cudaStream_t st) {
    UhcEngine *e = c->eng;
    const int E = c->E, nb = (E + 127) / 128;
    if (k.has_next && enqueue_push(c, R, c->d_next, k.has_mask ? c->d_mask : nullptr, st)) return -1;
    k_track_gate<<<nb, 128, 0, st>>>(R.istate, c->d_have, c->H, E, R.num_clips, c->d_status);
    CKT(cudaGetLastError());
    CKT(trackx::launch_obs(e, R.obs, st));
    std::string err;
    int rc = evalx::policy_enqueue(e, mlp, mcp, R.obs, k.log_std, (double *)k.zstats, k.zclip, c->d_ones, R.act, st, &err);
    if (rc) { g_tr_err = err; return rc; }
    if (uhc_env_step(e, R.act, nullptr, k.rew, R.cinfo, k.fail, R.end, R.pct, nullptr, st)) { g_tr_err = std::string("env step: ") + uhc_last_error(); return -1; }
    if (R.precision == 32)
        k_track_post<float><<<(E + 3) / 4, 128, 0, st>>>((const float *)R.state, R.istate, c->d_status, k.fail, k.fail_safe, E, c->d_steps, c->d_reseat, (float *)k.out);
    else
        k_track_post<double><<<(E + 3) / 4, 128, 0, st>>>((const double *)R.state, R.istate, c->d_status, k.fail, k.fail_safe, E, c->d_steps, c->d_reseat, (double *)k.out);
    CKT(cudaGetLastError());
    if (k.fail_safe) CKT(evalx::launch_reseat(e, E, c->d_reseat, st));
    return 0;
}

int track_step(UhcEngine *e, const double *next, const int *mask, const UhcMlp *mlp, const UhcMcp *mcp, const float *log_std, const double *zstats,
               float zclip, int fail_safe, void *out, float *rew, int *fail, void *stream) {
    const char *who = mcp ? "uhc_track_step_mcp" : "uhc_track_step";
    if (!e || (!mlp && !mcp) || !log_std || !zstats || !out || !rew || !fail) { g_tr_err = std::string(who) + ": null argument"; return -2; }
    TrackCtx *c = live_ctx(e, who);
    if (!c) return -2;
    unsigned long long sgen = 0; std::string err;
    int rc = evalx::policy_prepare(e, mlp, mcp, &sgen, &err);
    if (rc) { g_tr_err = err; return rc; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    cudaStream_t st = (cudaStream_t)stream;
    TrackKey key; memset(&key, 0, sizeof key);
    key.has_next = next != nullptr; key.has_mask = next && mask; key.fail_safe = fail_safe ? 1 : 0; key.zclip = zclip;
    key.scratch_gen = sgen; key.track_gen = c->gen; key.view_gen = R.view_gen; key.log_std = log_std; key.zstats = zstats;
    key.out = out; key.rew = rew; key.fail = fail;
    if (mcp) { key.nprim = mcp->nprim; for (int k = 0; k < mcp->nprim; k++) key.nets[k] = mcp->prim[k]; key.nets[mcp->nprim] = mcp->composer; }
    else key.nets[0] = *mlp;
    // the graphs hold the engine view, the policy scratch and the stream buffers as kernel parameters: a changed generation drops them
    for (size_t g = 0; g < c->graphs.size();) {
        const TrackKey &k = c->graphs[g].first;
        if (k.view_gen != key.view_gen || k.scratch_gen != key.scratch_gen || k.track_gen != key.track_gen) {
            cudaGraphExecDestroy(c->graphs[g].second); c->graphs.erase(c->graphs.begin() + g);
        } else g++;
    }
    // the caller's frames and mask are copied into the tracker's own buffers, so a new tensor per step replays the same graph
    if (next) CKT(cudaMemcpyAsync(c->d_next, next, (size_t)c->E * c->row_w * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (next && mask) CKT(cudaMemcpyAsync(c->d_mask, mask, (size_t)c->E * sizeof(int), cudaMemcpyDeviceToDevice, st));
    cudaGraphExec_t exec = nullptr;
    for (auto &g : c->graphs) if (g.first == key) { exec = g.second; break; }
    if (!exec) {
        cudaStream_t cs; CKT(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        cudaGraph_t graph = nullptr;
        CKT(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
        rc = enqueue_step(c, R, key, mlp, mcp, cs);
        cudaError_t ce = cudaStreamEndCapture(cs, &graph);
        cudaStreamDestroy(cs);
        if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (ce != cudaSuccess) { g_tr_err = std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce); return -1; }
        ce = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        CKT(ce);
        if (c->graphs.size() >= 32) { cudaGraphExecDestroy(c->graphs.front().second); c->graphs.erase(c->graphs.begin()); }
        c->graphs.emplace_back(key, exec);
    }
    CKT(cudaGraphLaunch(exec, st));
    return 0;
}

}  // namespace

extern "C" {

const char *uhc_track_last_error(void) { return g_tr_err.c_str(); }

int uhc_track_begin(UhcEngine *e, int window, int kind, int pose_dim, const int *fk_model_host, const double *shape_host) {
    if (!e) { g_tr_err = "uhc_track_begin: null engine"; return -2; }
    if (kind != UHC_MOTION_SMPL && kind != UHC_MOTION_QPOS) { g_tr_err = "uhc_track_begin: kind must be UHC_MOTION_SMPL or UHC_MOTION_QPOS"; return -2; }
    if (kind == UHC_MOTION_SMPL ? (pose_dim != 72 && pose_dim != 156) : pose_dim != UHC_NQ) { g_tr_err = "uhc_track_begin: pose_dim must be 72 or 156 (UHC_MOTION_SMPL) or 76 (UHC_MOTION_QPOS)"; return -2; }
    if (const char *why = trackx::cfg_error(e, window)) { g_tr_err = std::string("uhc_track_begin: ") + why; return -2; }
    const int E = uhc_num_envs(e);
    if (fk_model_host) for (int i = 0; i < E; i++) if (fk_model_host[i] < 0 || fk_model_host[i] >= trackx::num_shapes(e)) { g_tr_err = "uhc_track_begin: fk_model index out of range"; return -2; }
    if ((size_t)E * window * REC * 8 > ((size_t)1 << 40)) { g_tr_err = "uhc_track_begin: window too large"; return -2; }
    if (TrackCtx *old = find_ctx(e)) free_ctx(old);
    std::string err;
    if (trackx::install_table(e, window, fk_model_host, shape_host, &err)) { g_tr_err = err; return -1; }
    TrackCtx *c = new TrackCtx(); c->eng = e; g_tr.push_back(c);
    c->E = E; c->H = window; c->kind = kind; c->pose_dim = pose_dim; c->row_w = kind == UHC_MOTION_SMPL ? pose_dim + 3 : UHC_NQ;
    c->table_gen = trackx::table_gen(e); c->gen = ++g_tr_gen;
    const size_t En = E;
    CKT(cudaMalloc((void **)&c->d_raw, En * 2 * c->row_w * sizeof(double))); CKT(cudaMalloc((void **)&c->d_next, En * c->row_w * sizeof(double)));
    for (int **p : {&c->d_have, &c->d_steps, &c->d_dropped, &c->d_status, &c->d_reseat, &c->d_mask, &c->d_ids}) { CKT(cudaMalloc((void **)p, En * sizeof(int))); CKT(cudaMemset(*p, 0, En * sizeof(int))); }
    CKT(cudaMalloc((void **)&c->d_ones, En));
    k_fill_ones<<<(E + 255) / 256, 256>>>(c->d_ones, E);
    CKT(cudaGetLastError());
    if (fk_model_host) { CKT(cudaMalloc((void **)&c->d_fk, En * sizeof(int))); CKT(cudaMemcpy(c->d_fk, fk_model_host, En * sizeof(int), cudaMemcpyHostToDevice)); }
    CKT(cudaHostAlloc((void **)&c->h_ids, En * sizeof(int), cudaHostAllocDefault));
    CKT(cudaEventCreateWithFlags(&c->ids_done, cudaEventDisableTiming));
    CKT(cudaDeviceSynchronize());
    return 0;
}

int uhc_track_reset(UhcEngine *e, int n, const int *env_ids_host, const double *frames_dev, const float *qpos_dev, const float *qvel_dev, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_reset");
    if (!c) return -2;
    if (n < 1 || n > c->E || !env_ids_host || !frames_dev) { g_tr_err = "uhc_track_reset: needs 1 <= n <= E, env ids and frames"; return -2; }
    for (int i = 0; i < n; i++) if (env_ids_host[i] < 0 || env_ids_host[i] >= c->E) { g_tr_err = "uhc_track_reset: env id out of range"; return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    CKT(cudaEventSynchronize(c->ids_done));            // the previous reset's kernel has consumed the staging buffer
    memcpy(c->h_ids, env_ids_host, n * sizeof(int));
    CKT(cudaMemcpyAsync(c->d_ids, c->h_ids, n * sizeof(int), cudaMemcpyHostToDevice, st));
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    const MotionModel &m = trackx::motion_model(e);
    if (R.precision == 32)
        k_track_rows<float><<<(n + 127) / 128, 128, 0, st>>>(m, c->kind, c->pose_dim, c->row_w, c->H, n, c->d_ids, frames_dev, c->d_fk, (float *)R.expert,
                                                           c->d_raw, c->d_have, c->d_steps, c->d_dropped);
    else
        k_track_rows<double><<<(n + 127) / 128, 128, 0, st>>>(m, c->kind, c->pose_dim, c->row_w, c->H, n, c->d_ids, frames_dev, c->d_fk, (double *)R.expert,
                                                            c->d_raw, c->d_have, c->d_steps, c->d_dropped);
    CKT(cudaGetLastError());
    CKT(cudaEventRecord(c->ids_done, st));
    c->zeros.assign(n, 0); c->lens.assign(n, c->H);
    if (uhc_env_reset(e, n, env_ids_host, env_ids_host, c->zeros.data(), c->lens.data(), qpos_dev, qvel_dev, nullptr, stream)) {
        g_tr_err = std::string("uhc_track_reset: ") + uhc_last_error(); return -1;
    }
    return 0;
}

int uhc_track_step(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats,
                   float zclip, int fail_safe, void *state_out_dev, float *reward_dev, int *fail_dev, void *stream) {
    if (!mlp) { g_tr_err = "uhc_track_step: null policy"; return -2; }
    return track_step(e, next_frames_dev, mask_dev, mlp, nullptr, log_std, zfilter_stats, zclip, fail_safe, state_out_dev, reward_dev, fail_dev, stream);
}
int uhc_track_step_mcp(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats,
                       float zclip, int fail_safe, void *state_out_dev, float *reward_dev, int *fail_dev, void *stream) {
    if (!mcp) { g_tr_err = "uhc_track_step_mcp: null policy"; return -2; }
    return track_step(e, next_frames_dev, mask_dev, nullptr, mcp, log_std, zfilter_stats, zclip, fail_safe, state_out_dev, reward_dev, fail_dev, stream);
}

int uhc_track_push(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_push");
    if (!c) return -2;
    if (!next_frames_dev) { g_tr_err = "uhc_track_push: null frames"; return -2; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    return enqueue_push(c, R, next_frames_dev, mask_dev, (cudaStream_t)stream);
}

int uhc_track_obs(UhcEngine *e, float *obs_dev, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_obs");
    if (!c) return -2;
    if (!obs_dev) { g_tr_err = "uhc_track_obs: null output"; return -2; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = (c->E + 127) / 128;
    k_track_gate<<<nb, 128, 0, st>>>(R.istate, c->d_have, c->H, c->E, R.num_clips, c->d_status);
    CKT(cudaGetLastError());
    CKT(trackx::launch_obs(e, obs_dev, st));
    k_track_ungate<<<nb, 128, 0, st>>>(R.istate, c->d_status, c->E);
    CKT(cudaGetLastError());
    return 0;
}

int uhc_track_state(UhcEngine *e, int *out_host) {
    TrackCtx *c = e ? find_ctx(e) : nullptr;
    if (!c || !out_host) { g_tr_err = "uhc_track_state: not tracking or null output"; return -2; }
    const size_t E = c->E;
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    std::vector<int> steps(E), have(E), dropped(E), is(E * SI_SIZE);
    CKT(cudaDeviceSynchronize());
    CKT(cudaMemcpy(steps.data(), c->d_steps, E * sizeof(int), cudaMemcpyDeviceToHost));
    CKT(cudaMemcpy(have.data(), c->d_have, E * sizeof(int), cudaMemcpyDeviceToHost));
    CKT(cudaMemcpy(dropped.data(), c->d_dropped, E * sizeof(int), cudaMemcpyDeviceToHost));
    CKT(cudaMemcpy(is.data(), R.istate, E * SI_SIZE * sizeof(int), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < E; i++) {
        int *o = out_host + i * UHC_TRACK_STATE_COLS;
        o[0] = steps[i]; o[1] = is[i * SI_SIZE + SI_CUR_T]; o[2] = have[i]; o[3] = dropped[i];
    }
    return 0;
}

void uhc_track_end(UhcEngine *e) {
    if (TrackCtx *c = e ? find_ctx(e) : nullptr) free_ctx(c);
}

}  // extern "C"

bool uhc::trackx::tracking(UhcEngine *e) {
    const TrackCtx *c = e ? find_ctx(e) : nullptr;
    return c && trackx::table_gen(e) == c->table_gen;
}
