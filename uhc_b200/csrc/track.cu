// track.cu -- the batched physics tracker behind the C ABI (include/uhc_track.h): target frames streamed one per control step into a
// per-env window of expert-table rows, and one CUDA-graph replay (graph_cache.h) per step of
//   k_track_push  (when frames are passed)   per env: rebase a full window, the record of the new frame (track_core.h)
//   k_track_gate                             per env: an env whose row cur_t + 1 was never pushed gets an invalid record for this step
//   k_track_obs   (step_kernel.cu)           the observation of the stored state against row cur_t + 1 (track_obs.h)
//   ZFilter + policy GEMMs + mean action     uhc_eval_run's kernels (rollout.cu)
//   k_env_step                               unchanged, obs = null
//   k_track_post                             per env: the gated record restored, step count, fail_safe flag, the state gathered
//   k_eval_reseat (fail_safe only)           uhc_eval_run's re-seat on row cur_t
//
// Run-time subjects (uhc_track_set_subjects): k_subject (subject.cu) builds the bodies into a staging area, the host reads the inverted-body
// flags once, then k_subject_install writes each env's slot of the engine's tables (track_glue.h Slots) and points the env at it.
//
// Compiled on its own with -fmad=false (uhc_b200/build.py) like motion_lib.cu: the rows restate motion_lib.py's fp64 arithmetic and
// must equal uhc_load_motions' rows bit for bit.
#include <cuda_runtime.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_track.h"
#include "engine_slots.h"
#include "errors.h"
#include "eval_glue.h"
#include "graph_cache.h"
#include "track_glue.h"
#include "track_core.h"
#include "sim_core.h"
#include "subject_core.h"
#include "subject_glue.h"

using namespace uhc;

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

// one block per staged subject i: env ids[i]'s slot v = nshape + env of every table gets body i (the engine-precision tables rounded as
// uhc_engine_create's upload rounds, the FK table = body_f columns 0:6 as motion_body_table takes them), the env's clip model and FK variant
// become v, its shape row shape[i], and its record is invalidated until uhc_track_reset
template <class Real>
__global__ void k_subject_install(int n, const int *__restrict__ ids, int nshape, int nvert, const double *__restrict__ bf, const double *__restrict__ hull,
                                  const double *__restrict__ shape, Real *__restrict__ body_f, Real *__restrict__ hull_t, double *__restrict__ body6,
                                  double *__restrict__ hull64, int *__restrict__ clip_model, int *__restrict__ fk, Real *__restrict__ clip_shape,
                                  int *__restrict__ istate) {
    using subj::BODYF; using subj::NB;
    const int i = blockIdx.x, env = ids[i], v = nshape + env;
    const double *b = bf + (size_t)i * NB * BODYF, *h = hull + (size_t)i * nvert * 3;
    for (int k = threadIdx.x; k < NB * BODYF; k += blockDim.x) body_f[(size_t)v * NB * BODYF + k] = (Real)b[k];
    for (int k = threadIdx.x; k < NB * motion::BODY6; k += blockDim.x) body6[(size_t)v * NB * motion::BODY6 + k] = b[k / motion::BODY6 * BODYF + k % motion::BODY6];
    for (int k = threadIdx.x; k < nvert * 3; k += blockDim.x) { hull_t[(size_t)v * nvert * 3 + k] = (Real)h[k]; hull64[(size_t)env * nvert * 3 + k] = h[k]; }
    if (threadIdx.x < 17) clip_shape[(size_t)env * 17 + threadIdx.x] = (Real)shape[(size_t)i * 17 + threadIdx.x];
    if (threadIdx.x == 0) { clip_model[env] = v; fk[env] = v; istate[(size_t)env * SI_SIZE + SI_LEN] = 0; }
}

// every argument of a step that reaches a kernel; zeroed, then filled: its bytes are the graph's key
struct TrackKey {
    int has_next, has_mask, fail_safe; float zclip; evalx::Policy pol; const float *log_std; const double *zstats; void *out; float *rew; int *fail;
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
    GraphCache graphs{32};                         // one step each (graph_cache.h)
    // staging of uhc_track_set_subjects, grown to the largest call: betas [n][10], shape rows [n][17], built body_f / hull, flags, ids, genders
    double *d_sbeta = nullptr, *d_sshape = nullptr, *d_sbf = nullptr, *d_shull = nullptr; int *d_sbad = nullptr, *d_sids = nullptr, *d_sgender = nullptr;
    int s_cap = 0;
};
unsigned long long g_tr_gen = 0;                   // distinct per begin: graphs never outlive the buffers they hold

TrackCtx *find_ctx(UhcEngine *e) { return (TrackCtx *)engine_slot(e, SLOT_TRACK); }
void free_ctx(TrackCtx *c) {
    cudaDeviceSynchronize();
    c->graphs.clear();
    for (void *p : {(void *)c->d_raw, (void *)c->d_next, (void *)c->d_have, (void *)c->d_steps, (void *)c->d_dropped, (void *)c->d_status, (void *)c->d_reseat,
                    (void *)c->d_mask, (void *)c->d_fk, (void *)c->d_ids, (void *)c->d_ones, (void *)c->d_sbeta, (void *)c->d_sshape, (void *)c->d_sbf,
                    (void *)c->d_shull, (void *)c->d_sbad, (void *)c->d_sids, (void *)c->d_sgender}) if (p) cudaFree(p);
    if (c->h_ids) cudaFreeHost(c->h_ids);
    if (c->ids_done) cudaEventDestroy(c->ids_done);
    engine_slot(c->eng, SLOT_TRACK) = nullptr;
    delete c;
}

// the tracker of e while its table is still the engine's table and its cfg can run the stream, else null with the reason in uhc_err()
TrackCtx *live_ctx(UhcEngine *e, const char *who) {
    TrackCtx *c = e ? find_ctx(e) : nullptr;
    if (!c) { uhc_err() = std::string(who) + ": not tracking (uhc_track_begin)"; return nullptr; }
    if (trackx::table_gen(e) != c->table_gen) { uhc_err() = std::string(who) + ": tracking ended: the clip table was replaced"; return nullptr; }
    if (const char *why = trackx::cfg_error(e, c->H)) { uhc_err() = std::string(who) + ": " + why; return nullptr; }
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
    CK(cudaGetLastError());
    return 0;
}

int enqueue_step(TrackCtx *c, const evalx::EngineRefs &R, const TrackKey &k, cudaStream_t st) {
    UhcEngine *e = c->eng;
    const int E = c->E, nb = (E + 127) / 128;
    if (k.has_next && enqueue_push(c, R, c->d_next, k.has_mask ? c->d_mask : nullptr, st)) return -1;
    k_track_gate<<<nb, 128, 0, st>>>(R.istate, c->d_have, c->H, E, R.num_clips, c->d_status);
    CK(cudaGetLastError());
    CK(trackx::launch_obs(e, R.obs, st));
    const int rc = evalx::policy_enqueue(e, k.pol, R.obs, k.log_std, (double *)k.zstats, k.zclip, c->d_ones, R.act, st);
    if (rc) return rc;
    if (uhc_env_step(e, R.act, nullptr, k.rew, R.cinfo, k.fail, R.end, R.pct, nullptr, st)) return uhc_err_prefix("env step");
    if (R.precision == 32)
        k_track_post<float><<<(E + 3) / 4, 128, 0, st>>>((const float *)R.state, R.istate, c->d_status, k.fail, k.fail_safe, E, c->d_steps, c->d_reseat, (float *)k.out);
    else
        k_track_post<double><<<(E + 3) / 4, 128, 0, st>>>((const double *)R.state, R.istate, c->d_status, k.fail, k.fail_safe, E, c->d_steps, c->d_reseat, (double *)k.out);
    CK(cudaGetLastError());
    if (k.fail_safe) CK(evalx::launch_reseat(e, E, c->d_reseat, st));
    return 0;
}

int track_step(UhcEngine *e, const double *next, const int *mask, const UhcMlp *mlp, const UhcMcp *mcp, const float *log_std, const double *zstats,
               float zclip, int fail_safe, void *out, float *rew, int *fail, void *stream) {
    const char *who = mcp ? "uhc_track_step_mcp" : "uhc_track_step";
    if (!e || (!mlp && !mcp) || !log_std || !zstats || !out || !rew || !fail) { uhc_err() = std::string(who) + ": null argument"; return -2; }
    TrackCtx *c = live_ctx(e, who);
    if (!c) return -2;
    TrackKey k; memset(&k, 0, sizeof k);
    unsigned long long sgen = 0;
    int rc = evalx::policy_prepare(e, mlp, mcp, &k.pol, &sgen);
    if (rc) return rc;
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    cudaStream_t st = (cudaStream_t)stream;
    k.has_next = next != nullptr; k.has_mask = next && mask; k.fail_safe = fail_safe ? 1 : 0; k.zclip = zclip;
    k.log_std = log_std; k.zstats = zstats; k.out = out; k.rew = rew; k.fail = fail;
    std::string key; GraphCache::append(&key, &k);
    // the graphs also hold the policy scratch, the stream buffers and the engine view as kernel parameters: a changed generation drops them
    const GraphCache::Gens gens{sgen, c->gen, R.view_gen};
    c->graphs.drop_stale(gens);
    // the caller's frames and mask are copied into the tracker's own buffers, so a new tensor per step replays the same graph
    if (next) CK(cudaMemcpyAsync(c->d_next, next, (size_t)c->E * c->row_w * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (next && mask) CK(cudaMemcpyAsync(c->d_mask, mask, (size_t)c->E * sizeof(int), cudaMemcpyDeviceToDevice, st));
    cudaGraphExec_t exec = c->graphs.find(key);
    if (!exec) {
        rc = GraphCache::capture([&](cudaStream_t cs) { return enqueue_step(c, R, k, cs); }, &exec);
        if (rc) return rc;
        c->graphs.insert(std::move(key), gens, exec);
    }
    CK(cudaGraphLaunch(exec, st));
    return 0;
}

}  // namespace

extern "C" {

int uhc_track_begin(UhcEngine *e, int window, int kind, int pose_dim, const int *fk_model_host, const double *shape_host) {
    if (!e) { uhc_err() = "uhc_track_begin: null engine"; return -2; }
    if (kind != UHC_MOTION_SMPL && kind != UHC_MOTION_QPOS) { uhc_err() = "uhc_track_begin: kind must be UHC_MOTION_SMPL or UHC_MOTION_QPOS"; return -2; }
    if (kind == UHC_MOTION_SMPL ? (pose_dim != 72 && pose_dim != 156) : pose_dim != UHC_NQ) { uhc_err() = "uhc_track_begin: pose_dim must be 72 or 156 (UHC_MOTION_SMPL) or 76 (UHC_MOTION_QPOS)"; return -2; }
    if (const char *why = trackx::cfg_error(e, window)) { uhc_err() = std::string("uhc_track_begin: ") + why; return -2; }
    const int E = uhc_num_envs(e);
    if (fk_model_host) for (int i = 0; i < E; i++) if (fk_model_host[i] < 0 || fk_model_host[i] >= trackx::num_shapes(e)) { uhc_err() = "uhc_track_begin: fk_model index out of range"; return -2; }
    if ((size_t)E * window * REC * 8 > ((size_t)1 << 40)) { uhc_err() = "uhc_track_begin: window too large"; return -2; }
    if (TrackCtx *old = find_ctx(e)) free_ctx(old);
    if (trackx::install_table(e, window, fk_model_host, shape_host)) return -1;
    TrackCtx *c = new TrackCtx(); c->eng = e; engine_slot(e, SLOT_TRACK) = c;
    c->E = E; c->H = window; c->kind = kind; c->pose_dim = pose_dim; c->row_w = kind == UHC_MOTION_SMPL ? pose_dim + 3 : UHC_NQ;
    c->table_gen = trackx::table_gen(e); c->gen = ++g_tr_gen;
    const size_t En = E;
    CK(cudaMalloc((void **)&c->d_raw, En * 2 * c->row_w * sizeof(double))); CK(cudaMalloc((void **)&c->d_next, En * c->row_w * sizeof(double)));
    for (int **p : {&c->d_have, &c->d_steps, &c->d_dropped, &c->d_status, &c->d_reseat, &c->d_mask, &c->d_ids}) { CK(cudaMalloc((void **)p, En * sizeof(int))); CK(cudaMemset(*p, 0, En * sizeof(int))); }
    CK(cudaMalloc((void **)&c->d_ones, En));
    k_fill_ones<<<(E + 255) / 256, 256>>>(c->d_ones, E);
    CK(cudaGetLastError());
    if (fk_model_host || trackx::subject_builder(e)) {     // with run-time subjects every env's FK variant can change, at a fixed address
        CK(cudaMalloc((void **)&c->d_fk, En * sizeof(int)));
        if (fk_model_host) CK(cudaMemcpy(c->d_fk, fk_model_host, En * sizeof(int), cudaMemcpyHostToDevice));
        else CK(cudaMemset(c->d_fk, 0, En * sizeof(int)));
    }
    CK(cudaHostAlloc((void **)&c->h_ids, En * sizeof(int), cudaHostAllocDefault));
    CK(cudaEventCreateWithFlags(&c->ids_done, cudaEventDisableTiming));
    CK(cudaDeviceSynchronize());
    return 0;
}

int uhc_track_reset(UhcEngine *e, int n, const int *env_ids_host, const double *frames_dev, const float *qpos_dev, const float *qvel_dev, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_reset");
    if (!c) return -2;
    if (n < 1 || n > c->E || !env_ids_host || !frames_dev) { uhc_err() = "uhc_track_reset: needs 1 <= n <= E, env ids and frames"; return -2; }
    for (int i = 0; i < n; i++) if (env_ids_host[i] < 0 || env_ids_host[i] >= c->E) { uhc_err() = "uhc_track_reset: env id out of range"; return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaEventSynchronize(c->ids_done));            // the previous reset's kernel has consumed the staging buffer
    memcpy(c->h_ids, env_ids_host, n * sizeof(int));
    CK(cudaMemcpyAsync(c->d_ids, c->h_ids, n * sizeof(int), cudaMemcpyHostToDevice, st));
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    const MotionModel &m = trackx::motion_model(e);
    if (R.precision == 32)
        k_track_rows<float><<<(n + 127) / 128, 128, 0, st>>>(m, c->kind, c->pose_dim, c->row_w, c->H, n, c->d_ids, frames_dev, c->d_fk, (float *)R.expert,
                                                           c->d_raw, c->d_have, c->d_steps, c->d_dropped);
    else
        k_track_rows<double><<<(n + 127) / 128, 128, 0, st>>>(m, c->kind, c->pose_dim, c->row_w, c->H, n, c->d_ids, frames_dev, c->d_fk, (double *)R.expert,
                                                            c->d_raw, c->d_have, c->d_steps, c->d_dropped);
    CK(cudaGetLastError());
    CK(cudaEventRecord(c->ids_done, st));
    c->zeros.assign(n, 0); c->lens.assign(n, c->H);
    if (uhc_env_reset(e, n, env_ids_host, env_ids_host, c->zeros.data(), c->lens.data(), qpos_dev, qvel_dev, nullptr, stream)) return uhc_err_prefix("uhc_track_reset");
    return 0;
}

int uhc_track_step(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats,
                   float zclip, int fail_safe, void *state_out_dev, float *reward_dev, int *fail_dev, void *stream) {
    if (!mlp) { uhc_err() = "uhc_track_step: null policy"; return -2; }
    return track_step(e, next_frames_dev, mask_dev, mlp, nullptr, log_std, zfilter_stats, zclip, fail_safe, state_out_dev, reward_dev, fail_dev, stream);
}
int uhc_track_step_mcp(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats,
                       float zclip, int fail_safe, void *state_out_dev, float *reward_dev, int *fail_dev, void *stream) {
    if (!mcp) { uhc_err() = "uhc_track_step_mcp: null policy"; return -2; }
    return track_step(e, next_frames_dev, mask_dev, nullptr, mcp, log_std, zfilter_stats, zclip, fail_safe, state_out_dev, reward_dev, fail_dev, stream);
}

int uhc_track_push(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_push");
    if (!c) return -2;
    if (!next_frames_dev) { uhc_err() = "uhc_track_push: null frames"; return -2; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    return enqueue_push(c, R, next_frames_dev, mask_dev, (cudaStream_t)stream);
}

int uhc_track_obs(UhcEngine *e, float *obs_dev, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_obs");
    if (!c) return -2;
    if (!obs_dev) { uhc_err() = "uhc_track_obs: null output"; return -2; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = (c->E + 127) / 128;
    k_track_gate<<<nb, 128, 0, st>>>(R.istate, c->d_have, c->H, c->E, R.num_clips, c->d_status);
    CK(cudaGetLastError());
    CK(trackx::launch_obs(e, obs_dev, st));
    k_track_ungate<<<nb, 128, 0, st>>>(R.istate, c->d_status, c->E);
    CK(cudaGetLastError());
    return 0;
}

int uhc_track_state(UhcEngine *e, int *out_host) {
    TrackCtx *c = e ? find_ctx(e) : nullptr;
    if (!c || !out_host) { uhc_err() = "uhc_track_state: not tracking or null output"; return -2; }
    const size_t E = c->E;
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    std::vector<int> steps(E), have(E), dropped(E), is(E * SI_SIZE);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(steps.data(), c->d_steps, E * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(have.data(), c->d_have, E * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(dropped.data(), c->d_dropped, E * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(is.data(), R.istate, E * SI_SIZE * sizeof(int), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < E; i++) {
        int *o = out_host + i * UHC_TRACK_STATE_COLS;
        o[0] = steps[i]; o[1] = is[i * SI_SIZE + SI_CUR_T]; o[2] = have[i]; o[3] = dropped[i];
    }
    return 0;
}

void uhc_track_end(UhcEngine *e) {
    if (TrackCtx *c = e ? find_ctx(e) : nullptr) free_ctx(c);
}

int uhc_track_graph_count(const UhcEngine *e) {
    const TrackCtx *c = e ? (const TrackCtx *)engine_slot(e, SLOT_TRACK) : nullptr;
    return c ? (int)c->graphs.size() : 0;
}

int uhc_track_subjects_enable(UhcEngine *e, const UhcSubjectBasis *basis) {
    if (!e || !basis) { uhc_err() = "uhc_track_subjects_enable: null argument"; return -2; }
    if (trackx::tracking(e)) { uhc_err() = "uhc_track_subjects_enable: tracking is active (call it before uhc_track_begin, or after uhc_track_end)"; return -2; }
    const UhcModelHost base = trackx::base_model(e);
    subjx::Builder *b = nullptr;
    if (const int rc = subjx::builder_create(&base, basis, "uhc_track_subjects_enable", &b)) return rc;
    return trackx::enable_subjects(e, b);
}

int uhc_track_subject_tables(UhcEngine *e, int env, double *body_f_host, double *hull_host, double *fk_body_host, double *hull64_host) {
    if (!e || !trackx::subject_builder(e)) { uhc_err() = "uhc_track_subject_tables: run-time subjects are not enabled"; return -2; }
    if (env < 0 || env >= uhc_num_envs(e)) { uhc_err() = "uhc_track_subject_tables: env id out of range"; return -2; }
    trackx::Slots s; trackx::slots(e, &s);
    const size_t v = (size_t)s.nshape + env, nb = (size_t)subj::NB * subj::BODYF, nh = (size_t)s.nvert * 3, rs = s.precision == 32 ? 4 : 8;
    std::vector<unsigned char> tmp(nh * rs);
    auto widen = [&](const void *src, size_t n, double *out) -> int {
        CK(cudaMemcpy(tmp.data(), src, n * rs, cudaMemcpyDeviceToHost));
        for (size_t k = 0; k < n; k++) out[k] = rs == 4 ? (double)((const float *)tmp.data())[k] : ((const double *)tmp.data())[k];
        return 0;
    };
    CK(cudaDeviceSynchronize());
    if (body_f_host && widen((const char *)s.body_f + v * nb * rs, nb, body_f_host)) return -1;
    if (hull_host && widen((const char *)s.hull + v * nh * rs, nh, hull_host)) return -1;
    if (fk_body_host) CK(cudaMemcpy(fk_body_host, s.body6 + v * subj::NB * motion::BODY6, (size_t)subj::NB * motion::BODY6 * sizeof(double), cudaMemcpyDeviceToHost));
    if (hull64_host) CK(cudaMemcpy(hull64_host, s.hull64 + (size_t)env * nh, nh * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
}

int uhc_track_set_subjects(UhcEngine *e, int n, const int *env_ids_host, const double *shape_host, void *stream) {
    TrackCtx *c = live_ctx(e, "uhc_track_set_subjects");
    if (!c) return -2;
    const subjx::Builder *b = trackx::subject_builder(e);
    if (!b) { uhc_err() = "uhc_track_set_subjects: run-time subjects are not enabled (uhc_track_subjects_enable before uhc_track_begin)"; return -2; }
    if (n < 1 || n > c->E || !env_ids_host || !shape_host) { uhc_err() = "uhc_track_set_subjects: needs 1 <= n <= E, env ids and shape rows"; return -2; }
    std::vector<char> seen(c->E, 0);
    std::vector<double> beta((size_t)n * subj::NBETA);
    std::vector<int> gender(n);
    for (int i = 0; i < n; i++) {
        const int env = env_ids_host[i];
        if (env < 0 || env >= c->E || seen[env]) { uhc_err() = "uhc_track_set_subjects: env id out of range or listed twice"; return -2; }
        seen[env] = 1;
        const double *r = shape_host + (size_t)i * 17;
        for (int k = 0; k < 17; k++)
            if (!isfinite(r[k])) { uhc_err() = "uhc_track_set_subjects: row " + std::to_string(i) + ": non-finite beta or gender"; return -2; }
        const double g = r[16];
        if (!(g == 0.0 || g == 1.0 || g == 2.0) || !subjx::has_gender(b, (int)g)) {
            uhc_err() = "uhc_track_set_subjects: row " + std::to_string(i) + ": gender code " + std::to_string(g) + " has no basis"; return -2;
        }
        gender[i] = (int)g;
        for (int l = 0; l < subj::NBETA; l++) beta[(size_t)i * subj::NBETA + l] = r[l];
    }
    const int V = subjx::nvert(b);
    if (c->s_cap < n) {
        for (void *p : {(void *)c->d_sbeta, (void *)c->d_sshape, (void *)c->d_sbf, (void *)c->d_shull, (void *)c->d_sbad, (void *)c->d_sids, (void *)c->d_sgender}) if (p) cudaFree(p);
        c->d_sbeta = c->d_sshape = c->d_sbf = c->d_shull = nullptr; c->d_sbad = c->d_sids = c->d_sgender = nullptr; c->s_cap = 0;
        const size_t N = n;
        CK(cudaMalloc((void **)&c->d_sbeta, N * subj::NBETA * sizeof(double))); CK(cudaMalloc((void **)&c->d_sshape, N * 17 * sizeof(double)));
        CK(cudaMalloc((void **)&c->d_sbf, N * subj::NB * subj::BODYF * sizeof(double))); CK(cudaMalloc((void **)&c->d_shull, N * V * 3 * sizeof(double)));
        for (int **p : {&c->d_sbad, &c->d_sids, &c->d_sgender}) CK(cudaMalloc((void **)p, N * sizeof(int)));
        c->s_cap = n;
    }
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemcpyAsync(c->d_sbeta, beta.data(), beta.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(c->d_sgender, gender.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(c->d_sshape, shape_host, (size_t)n * 17 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(c->d_sids, env_ids_host, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(subjx::launch(b, n, c->d_sbeta, c->d_sgender, c->d_sbf, c->d_shull, c->d_sbad, st));
    std::vector<int> bad(n);
    CK(cudaMemcpyAsync(bad.data(), c->d_sbad, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));         // the one synchronise: an inverted body is refused before any table is written
    for (int i = 0; i < n; i++)
        if (bad[i]) {
            uhc_err() = "uhc_track_set_subjects: row " + std::to_string(i) + ": the map of body " + std::to_string(bad[i] - 1) + " inverts it (det A <= 0)";
            return -2;
        }
    trackx::Slots s; trackx::slots(e, &s);
    if (s.precision == 32)
        k_subject_install<float><<<n, 256, 0, st>>>(n, c->d_sids, s.nshape, s.nvert, c->d_sbf, c->d_shull, c->d_sshape, (float *)s.body_f, (float *)s.hull,
                                                     s.body6, s.hull64, s.clip_model, c->d_fk, (float *)s.shape, s.istate);
    else
        k_subject_install<double><<<n, 256, 0, st>>>(n, c->d_sids, s.nshape, s.nvert, c->d_sbf, c->d_shull, c->d_sshape, (double *)s.body_f, (double *)s.hull,
                                                      s.body6, s.hull64, s.clip_model, c->d_fk, (double *)s.shape, s.istate);
    CK(cudaGetLastError());
    return 0;
}

}  // extern "C"

bool uhc::trackx::tracking(UhcEngine *e) {
    const TrackCtx *c = e ? find_ctx(e) : nullptr;
    return c && trackx::table_gen(e) == c->table_gen;
}
