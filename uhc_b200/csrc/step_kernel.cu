// step_kernel.cu -- CUDA kernels + C ABI (include/uhc_b200.h) for the batched humanoid env: one warp per environment,
// working set in shared memory, state records in HBM.  sm_90a.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../include/uhc_rollout.h"
#include "env_step.h"
#include "errors.h"
#include "motion_core.h"
#include "eval_glue.h"
#include "curriculum_core.h"
#include "track_obs.h"
#include "track_glue.h"
#include "subject_glue.h"

using namespace uhc;

// the small per-model tables every solve walks (joint gains / armature, tree-level table) are staged once per CTA behind the
// EPB work sets; the Model is pointed at the copies (sim_core.h reads them with shared-space loads)
template <class Real, int EPB>
__device__ __forceinline__ void stage_tables(EngineView<Real> &ev, unsigned char *smem) {
    Real *s_dof = reinterpret_cast<Real *>(smem + EPB * sizeof(Work<Real>));
    Real *s_lim = s_dof + NV * 4;
    int *s_lvl = reinterpret_cast<int *>(s_lim + NV * 4);
    for (int i = threadIdx.x; i < NV * 4; i += blockDim.x) { s_dof[i] = ev.model.dof_f[i]; s_lim[i] = ev.model.dof_lim[i]; }
    for (int i = threadIdx.x; i < (MAXLEVEL + 1) * LVL_G; i += blockDim.x) s_lvl[i] = ev.model.lvl_pack[i];
    LaneTopo *s_topo = reinterpret_cast<LaneTopo *>(s_lvl + (MAXLEVEL + 1) * LVL_G);
    if (threadIdx.x < 32) s_topo[threadIdx.x] = lane_topo(ev.model, (int)threadIdx.x);
    __syncthreads();
    ev.model.dof_f = s_dof; ev.model.dof_lim = s_lim; ev.model.lvl_pack = s_lvl; ev.model.topo_s = s_topo;
}

// warps per substep alignment group (sim_core.h, UHC_CTA_SYNC): the fp32 kernel's 16-warp CTA is two groups, the fp64 kernel's one
constexpr int SYNC_GROUP = 8;
#ifdef UHC_MAXNREG     /* experiment knob: cap registers without changing the CTA shape */
#define UHC_STEP_BOUNDS(EPB, Real) __maxnreg__(UHC_MAXNREG)
#else
#define UHC_STEP_BOUNDS(EPB, Real) __launch_bounds__(32 * EPB, 1)
#endif
template <class Real, int EPB, bool CUR = false>
__global__ void UHC_STEP_BOUNDS(EPB, Real)
k_env_step(EngineView<Real> ev, const float *__restrict__ act, float *__restrict__ obs, float *__restrict__ rew, float *__restrict__ cinfo,
           int *__restrict__ fail, int *__restrict__ end, float *__restrict__ pct, float *__restrict__ torque, const int *__restrict__ order) {
    extern __shared__ __align__(16) unsigned char smem[];
    constexpr int NGRP = (EPB + SYNC_GROUP - 1) / SYNC_GROUP;
    __shared__ int s_nvalid[NGRP];
    const int warp = threadIdx.x >> 5, slot = blockIdx.x * EPB + warp, grp = warp / SYNC_GROUP;
    if (threadIdx.x < NGRP) s_nvalid[threadIdx.x] = 0;
    stage_tables<Real, EPB>(ev, smem);
    // the warps of an alignment group wait for each other every substep: `order` groups environments that needed a similar number of
    // solver iterations in the previous step into the same CTA (k_order_envs), outputs stay indexed by the environment id
    const int env = slot < ev.num_envs ? (order ? order[slot] : slot) : -1;
    const bool valid = env >= 0 && env_record_valid(ev, env);
    if (valid && (threadIdx.x & 31) == 0) atomicAdd(&s_nvalid[grp], 1);
    __syncthreads();
    if (!valid) {   // no work (grid tail) or a stale / never-reset env record: flagged outputs, and the warp is not counted in the substep barrier
        if (env >= 0) env_step_invalid<Real, float>(ev, obs ? obs + (size_t)env * ev.cfg.obs_dim : nullptr, rew ? rew + env : nullptr, cinfo ? cinfo + (size_t)env * 5 : nullptr,
                                                    fail ? fail + env : nullptr, end ? end + env : nullptr, pct ? pct + env : nullptr);
        return;
    }
    Work<Real> &w = reinterpret_cast<Work<Real> *>(smem)[warp];
    if ((threadIdx.x & 31) == 0) { w.sync_threads = 32 * s_nvalid[grp]; w.sync_id = 1 + grp; }
    state_mbar_init(w);            // mbarrier of this warp's bulk-async (TMA) state load
    env_step_warp<Real, float, CUR>(ev, env, w, act + (size_t)env * ev.cfg.act_dim, obs ? obs + (size_t)env * ev.cfg.obs_dim : nullptr, rew ? rew + env : nullptr,
                               cinfo ? cinfo + (size_t)env * 5 : nullptr, fail ? fail + env : nullptr, end ? end + env : nullptr,
                               pct ? pct + env : nullptr, torque ? torque + (size_t)env * NSUB * NU : nullptr);
}

// counting sort of the environments by the Newton iterations of their previous step (one block)
__global__ void __launch_bounds__(1024) k_order_envs(const int *__restrict__ istate, int E, int *__restrict__ order) {
    __shared__ int hist[64], base[64];
    if (threadIdx.x < 64) hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < E; i += blockDim.x) { int k = istate[(size_t)i * SI_SIZE + SI_NEWTON]; k = k < 0 ? 0 : (k > 63 ? 63 : k); atomicAdd(&hist[k], 1); }
    __syncthreads();
    if (threadIdx.x == 0) { int run = 0; for (int k = 0; k < 64; k++) { base[k] = run; run += hist[k]; } }
    __syncthreads();
    for (int i = threadIdx.x; i < E; i += blockDim.x) { int k = istate[(size_t)i * SI_SIZE + SI_NEWTON]; k = k < 0 ? 0 : (k > 63 ? 63 : k); order[atomicAdd(&base[k], 1)] = i; }
}

template <class Real, int EPB>
__global__ void __launch_bounds__(32 * EPB)
k_env_reset(EngineView<Real> ev, int n, const int *__restrict__ ids, const int *__restrict__ clip, const int *__restrict__ start,
            const int *__restrict__ len, const float *__restrict__ qpos, const float *__restrict__ qvel, float *__restrict__ obs) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int warp = threadIdx.x >> 5, i = blockIdx.x * EPB + warp;
    stage_tables<Real, EPB>(ev, smem);
    if (i >= n) return;
    Work<Real> &w = reinterpret_cast<Work<Real> *>(smem)[warp];
    const int env = ids[i];
    // optional overrides arrive as float; stage them through the work set's scratch vectors
    Real *qo = nullptr, *vo = nullptr;
    if (qpos) { qo = w.as_; vo = w.Mp; const int lane = threadIdx.x & 31;   // vectors untouched before the reset copies them out
        for (int k = lane; k < NQ; k += 32) qo[k] = (Real)qpos[(size_t)i * NQ + k];
        for (int k = lane; k < NV; k += 32) vo[k] = qvel ? (Real)qvel[(size_t)i * NV + k] : Real(0);
        __syncwarp(); }
    env_reset_warp<Real, float>(ev, env, w, clip[i], start[i], len[i], qo, vo, obs ? obs + (size_t)env * ev.cfg.obs_dim : nullptr);
}

// device evaluation's fail_safe (eval.cu): the re-seat of uhc_env_set_state_batch -- k_save_restore_bquat, k_env_reset with the
// fp32-rounded expert qpos / qvel of frame min(cur_t, len - 1) as override and no obs, k_save_restore_bquat -- in one launch, for the
// envs i < n whose flag is set (the flag is written on the device by k_eval_frame, so the graph replays need no host decision)
template <class Real, int EPB>
__global__ void __launch_bounds__(32 * EPB)
k_eval_reseat(EngineView<Real> ev, int n, const int *__restrict__ reseat) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int warp = threadIdx.x >> 5, env = blockIdx.x * EPB + warp, lane = threadIdx.x & 31;
    const bool mine = env < n && reseat[env] != 0;
    if (!__syncthreads_or(mine)) return;      // most steps re-seat no env of the block: skip the table staging (uniform per block)
    stage_tables<Real, EPB>(ev, smem);
    if (!mine) return;
    Work<Real> &w = reinterpret_cast<Work<Real> *>(smem)[warp];
    int *is = ev.istate + (size_t)env * SI_SIZE;
    const int cur_t = is[SI_CUR_T], clip = is[SI_CLIP], start = is[SI_START], len = is[SI_LEN];
    Real *bq = ev.state + (size_t)env * ST_SIZE + ST_BQUAT;       // bquat + pbquat: 192 Reals, 6 per lane
    Real keep[6];
    for (int k = 0; k < 6; k++) keep[k] = bq[lane + 32 * k];
    const Real *f = expert_frame(ev, clip, start, len, cur_t);
    Real *qo = w.as_, *vo = w.Mp;                                  // the override's staging vectors of k_env_reset
    for (int k = lane; k < NQ; k += 32) qo[k] = (Real)(float)f[EX_QPOS + k];
    for (int k = lane; k < NV; k += 32) vo[k] = (Real)(float)f[EX_QVEL + k];
    __syncwarp();
    env_reset_warp<Real, float>(ev, env, w, clip, start, len, qo, vo, (float *)nullptr);
    __syncwarp();
    for (int k = 0; k < 6; k++) bq[lane + 32 * k] = keep[k];
    if (lane == 0) is[SI_CUR_T] = cur_t;
}

// the tracker's observation pass (track.cu): one warp per env, the observation of its stored state against row cur_t + 1 through the step
// kernel's write_obs (track_obs.h); an env the step kernel will skip (invalid record, or a missing row: track.cu gates it) gets a zero row
constexpr int EPB_OBS = 2;
template <class Real>
__global__ void __launch_bounds__(32 * EPB_OBS) k_track_obs(EngineView<Real> ev, float *__restrict__ obs) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int warp = threadIdx.x >> 5, env = blockIdx.x * EPB_OBS + warp, lane = threadIdx.x & 31;
    if (env >= ev.num_envs) return;
    float *o = obs + (size_t)env * ev.cfg.obs_dim;
    if (!env_record_valid(ev, env)) { for (int i = lane; i < ev.cfg.obs_dim; i += 32) o[i] = 0.f; return; }
    Work<Real> &w = reinterpret_cast<Work<Real> *>(smem)[warp];
    track_obs_warp<Real, float>(ev, env, w, o);
}

// uhc_curriculum_reseed: the re-seed draw of the step kernel for every env (one thread each); the resets follow as k_env_reset
template <class Real>
__global__ void k_cur_sample(EngineView<Real> ev, int *__restrict__ out) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= ev.num_envs) return;
    int *is = ev.istate + (size_t)env * SI_SIZE;
    const int episode = is[SI_EPISODE] + 1;
    int c, st, ln;
    sample_clip_cur(ev, env, episode, &c, &st, &ln);
    is[SI_EPISODE] = episode;
    const int E = ev.num_envs;
    out[env] = env; out[E + env] = c; out[2 * E + env] = st; out[3 * E + env] = ln;
}

// parity / evaluation hook: gather q, v, xpos, bquat (+ the integer record) of the listed envs into one staging array
template <class Real>
__global__ void k_gather_state(const Real *__restrict__ state, const int *__restrict__ istate, const int *__restrict__ ids, int n, double *__restrict__ out, int *__restrict__ iout) {
    const int i = blockIdx.x; if (i >= n) return;
    const int env = ids[i];
    const Real *st = state + (size_t)env * ST_SIZE;
    double *o = out + (size_t)i * 319;
    for (int k = threadIdx.x; k < NQ; k += blockDim.x) o[k] = (double)st[ST_Q + k];
    for (int k = threadIdx.x; k < NV; k += blockDim.x) o[76 + k] = (double)st[ST_V + k];
    for (int k = threadIdx.x; k < 72; k += blockDim.x) o[151 + k] = (double)st[ST_XPOS + k];
    for (int k = threadIdx.x; k < 96; k += blockDim.x) o[223 + k] = (double)st[ST_BQUAT + k];
    if (threadIdx.x < SI_SIZE) iout[(size_t)i * SI_SIZE + threadIdx.x] = istate[(size_t)env * SI_SIZE + threadIdx.x];
}
// set_state keeps cur_t and the body quaternions of the env (humanoid_im.py:902-905 only overwrites qpos / qvel)
template <class Real>
__global__ void k_save_restore_bquat(Real *__restrict__ state, int *__restrict__ istate, const int *__restrict__ ids, int n, Real *__restrict__ keep, int *__restrict__ keep_t, int restore) {
    const int i = blockIdx.x; if (i >= n) return;
    const int env = ids[i];
    Real *st = state + (size_t)env * ST_SIZE + ST_BQUAT;
    for (int k = threadIdx.x; k < 192; k += blockDim.x) { if (restore) st[k] = keep[(size_t)i * 192 + k]; else keep[(size_t)i * 192 + k] = st[k]; }
    if (threadIdx.x == 0) { if (restore) istate[(size_t)env * SI_SIZE + SI_CUR_T] = keep_t[i]; else keep_t[i] = istate[(size_t)env * SI_SIZE + SI_CUR_T]; }
}

struct UhcEngine {
    int E, device, precision, launches;
    std::vector<void *> allocs;
    EngineView<float> evf; EngineView<double> evd;
    int *d_clip_model = nullptr; int nshape = 1;
    void *d_expert = nullptr, *d_shape = nullptr; int *d_clip_adr = nullptr; float *d_clip_cdf = nullptr; int num_clips = 0;
    // staging for the host-buffer API
    float *d_act = nullptr, *d_obs = nullptr, *d_rew = nullptr, *d_cinfo = nullptr, *d_pct = nullptr; int *d_fail = nullptr, *d_end = nullptr;
    int *d_ids = nullptr; int ids_cap = 0;
    int *h_ids = nullptr;                 // pinned host staging of the reset arguments (ids, clip, start, len)
    cudaEvent_t ids_done = nullptr;       // the last reset kernel that read d_ids has been enqueued before this event
    float *d_qv = nullptr; int qv_cap = 0; void *d_keep = nullptr; int *d_keep_t = nullptr;   // set_state staging: [n][76+75] floats, kept bquat / cur_t
    double *d_gather = nullptr; int *d_gather_i = nullptr; int gather_cap = 0;
    std::vector<float> clip_w;            // clip sampling weights behind clip_cdf (uhc_set_clip_weights), empty = sample_keys rule
    int *d_order = nullptr;   // warp slot -> environment (work-sorted each step), null = identity
    std::vector<int> clip_len_h;   // host copy of the clip lengths (argument validation)
    std::vector<int> clip_adr_h;   // host copy of the first frame of every clip
    // bumped whenever anything a launch captures by value changes: the EngineView (cfg, clip table / model / CDF / neutral pointers).
    // CUDA graphs of the device evaluation (eval.cu) are keyed on it, so a table load or set_cfg never replays stale parameters
    unsigned long long view_gen = 0;
    unsigned long long table_gen = 0;   // bumped with every clip-table replacement: a tracker (track.cu) owns the table it installed only
    motion::MotionModel mo_model;  // FK tables of the device motion library (uhc_load_motions); mo_model.body = fp64 offsets / ipos on the device
    float mo_ms[2] = {0.f, 0.f};   // kernel / row-copy time of the last uhc_load_motions (CUDA events, ms)
    // device curriculum (uhc_curriculum_*): off while cur.M == 0.  cur_gen changes with everything the sampler reads of it by value
    cur::Dev cur = {};
    float prec_freq = 0.f; int fit_clip = -1;
    unsigned long long cur_gen = 0;
    size_t cur_cnt_cap = 0, cur_rank_cap = 0;
    int *d_reseed = nullptr;       // [4][E] ids / clip / start / len of uhc_curriculum_reseed
    int *d_push = nullptr; int push_cap = 0;   // [3][n] clip / percent bits / start of uhc_curriculum_push
    // variant 0 of the model in fp64 on the host: the base of the run-time subject builder
    std::vector<double> base_bf, base_hull, base_dof; std::vector<int> base_hull_adr, base_hull_num, base_parent, base_sub_end;
    // run-time subjects (uhc_track_subjects_enable): nslot = E once enabled, and variant nshape + env of body_f / hull / mo_model.body is env's
    // own body; d_slot_hull holds the same hulls in fp64 ([E][nvert][3], the floor measurements' vertices)
    subjx::Builder *subj = nullptr; int nslot = 0;
    double *d_slot_hull = nullptr;
};

template <class T> static int dev_copy(UhcEngine *e, T **dst, const T *src, size_t n) {
    CK(cudaMalloc((void **)dst, n * sizeof(T))); e->allocs.push_back(*dst);
    CK(cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}
template <class Real> static int dev_copy_real(UhcEngine *e, const Real **dst, const double *src, size_t n) {
    std::vector<Real> tmp(n); for (size_t i = 0; i < n; i++) tmp[i] = (Real)src[i];
    Real *d; if (dev_copy(e, &d, tmp.data(), n)) return -1; *dst = d; return 0;
}
template <class Real> static void fill_cfg(EnvCfg<Real> &c, const UhcEnvCfg *h) {
    for (int i = 0; i < 4; i++) c.base_rot[i] = (Real)h->base_rot[i];
    c.rfc_scale = (Real)h->rfc_scale; c.rfc_lim = (Real)h->rfc_lim; c.rfc_rate = (Real)h->rfc_rate; c.body_diff_thresh = (Real)h->body_diff_thresh;
    c.meta_pd = h->meta_pd; c.env_episode_len = h->env_episode_len; c.trail_steps = h->trail_steps; c.newton_max_iter = h->newton_max_iter;
    for (int i = 0; i < 5; i++) { c.w[i] = (Real)h->w[i]; c.k[i] = (Real)h->k[i]; }
    c.newton_tol = (Real)h->newton_tol;
    c.auto_reset = h->auto_reset; c.t_min = h->t_min; c.t_max = h->t_max; c.reset_seed = h->reset_seed;
    c.reactive_v = h->reactive_v; c.reactive_rate = (Real)h->reactive_rate;
    c.rfc_mode = (h->rfc_mode == 1 || h->rfc_mode == 2) ? h->rfc_mode : 0; c.vf_dim = c.rfc_mode == 1 ? VF_BODY_DIM * NB : (c.rfc_mode == 2 ? 0 : 6); c.act_dim = NU + c.vf_dim + (h->meta_pd ? 2 * NSUB : 0);
    for (int b = 0; b < NB; b++) c.vf_slot[b] = (signed char)((h->vf_slot[b] >= 0 && h->vf_slot[b] < NB) ? h->vf_slot[b] : b);
    c.obs_v = (h->obs_v == 1 || h->obs_v == 3 || h->obs_v == 5 || h->obs_v == 6) ? h->obs_v : 2;
    c.fut_frames = h->fut_frames > 0 ? h->fut_frames : 10; c.fut_skip = h->fut_skip > 0 ? h->fut_skip : 10;     // cc_cfg.get("fut_frames", 10), get("skip", 10)
    c.has_shape = h->no_shape ? 0 : 1; c.obs_block = c.has_shape ? OBS_DIM : OBS_DIM - 17;
    c.obs_dim = c.obs_v == 1 ? OBS_DIM_V1 : (c.obs_v == 3 ? c.obs_block * c.fut_frames : c.obs_block);
    if (c.obs_v == 5 || c.obs_v == 6) c.obs_dim = (c.obs_v == 5 ? 636 : 384) + (c.has_shape ? 17 : 0);      // get_full_obs_v5 / v6
    c.term_body = (h->term_body == 1 || h->term_body == 2) ? h->term_body : 0; c.head_body = (h->head_body >= 0 && h->head_body < NB) ? h->head_body : 13;
    c.reward_mul = h->reward_mul ? 1 : 0;
}
template <class Real> static int build_view(UhcEngine *e, EngineView<Real> &ev, const UhcModelHost *m, const UhcEnvCfg *cfg) {
    Model<Real> &M = ev.model;
    const int nshape = m->nshape > 0 ? m->nshape : 1;
    if (dev_copy_real<Real>(e, &M.body_f, m->body_f, (size_t)nshape * NB * BODYF) || dev_copy_real<Real>(e, &M.dof_f, m->dof_f, NV * 4) ||
        dev_copy_real<Real>(e, &M.hull, m->hull, (size_t)nshape * m->nvert * 3)) return -1;
    M.nshape = nshape; M.nvert = m->nvert; M.topo_s = nullptr;
    {   // joint limits: without a table every hinge is unlimited
        std::vector<double> lim(NV * 4, 0.0);
        for (int i = 0; i < NV; i++) { lim[4 * i] = -1e30; lim[4 * i + 1] = 1e30; lim[4 * i + 2] = 1.0; }
        if (dev_copy_real<Real>(e, &M.dof_lim, m->dof_lim ? m->dof_lim : lim.data(), NV * 4)) return -1;
    }
    int *p;
#define CPI(field, n) do { if (dev_copy(e, &p, m->field, (size_t)(n))) return -1; M.field = p; } while (0)
    CPI(hull_adr, NB); CPI(hull_num, NB); CPI(nbr, m->nnbr); CPI(nbradr, m->nvert + 1); CPI(parent, NB); CPI(depth, NB); CPI(child_adr, NB + 1);
    CPI(child, NB - 1); CPI(body_sub_end, NB); CPI(ee, 5); CPI(lvl_tab, (MAXLEVEL + 1) * LVL_G * 5); CPI(lvl_pack, (MAXLEVEL + 1) * LVL_G);
#undef CPI
    M.dt = (Real)m->dt; M.margin = (Real)m->margin; M.mu = (Real)m->mu; M.solref0 = (Real)m->solref[0]; M.solref1 = (Real)m->solref[1];
    M.simp0 = (Real)m->solimp[0]; M.simp1 = (Real)m->solimp[1]; M.simp2 = (Real)m->solimp[2]; M.simp3 = (Real)m->solimp[3]; M.simp4 = (Real)m->solimp[4];
    M.gravz = (Real)m->gravz;
    fill_cfg(ev.cfg, cfg);
    ev.num_envs = e->E;
    Real *st; CK(cudaMalloc((void **)&st, (size_t)e->E * ST_SIZE * sizeof(Real))); e->allocs.push_back(st);
    CK(cudaMemset(st, 0, (size_t)e->E * ST_SIZE * sizeof(Real)));
    int *is; CK(cudaMalloc((void **)&is, (size_t)e->E * SI_SIZE * sizeof(int))); e->allocs.push_back(is);
    CK(cudaMemset(is, 0, (size_t)e->E * SI_SIZE * sizeof(int)));
    int *cn; CK(cudaMalloc((void **)&cn, 4 * sizeof(int))); e->allocs.push_back(cn); CK(cudaMemset(cn, 0, 4 * sizeof(int)));
    ev.counters = cn; ev.neutral = nullptr;
    int *el; CK(cudaMalloc((void **)&el, (size_t)e->E * 3 * sizeof(int))); e->allocs.push_back(el); CK(cudaMemset(el, 0xFF, (size_t)e->E * 3 * sizeof(int)));
    ev.ep_log = el; ev.ep_start_log = el + (size_t)2 * e->E;
    ev.cur.pct = nullptr; ev.cur.start = nullptr; ev.cur.meta = nullptr; ev.cur.max_freq = 0; ev.cur.fit_clip = -1; ev.cur.prec_freq = 0.f;
    ev.state = st; ev.istate = is; ev.expert = nullptr; ev.clip_adr = nullptr; ev.clip_shape = nullptr; ev.clip_model = nullptr; ev.clip_cdf = nullptr;
#ifdef UHC_PHASE_CLOCKS
    ev.phase_cyc = nullptr;
#endif
    return 0;
}

// environments (warps) per block.  fp32: one 16-warp CTA per SM, so 132 SMs hold 2112 envs and 4096 envs run in two full waves
// (at 14 per SM they took three, the last one a 58-CTA tail)
constexpr int EPB_F = 16, EPB_D = 2;
template <class Real, int EPB> constexpr size_t step_smem() { return EPB * sizeof(Work<Real>) + 2 * NV * 4 * sizeof(Real) + (MAXLEVEL + 1) * LVL_G * sizeof(int) + 32 * sizeof(LaneTopo); }
// sm_90: 228 KiB of shared memory per SM, 1 KiB of it reserved per block, 32 B of static shared memory here (64 allowed).  A few hundred bytes
// more in Work / LaneTopo and the 16-warp block no longer launches, so it is a compile-time error
static_assert(step_smem<float, EPB_F>() + 1024 + 64 <= 228 * 1024, "k_env_step<float>: the 16 work sets of a block no longer fit one SM");

extern "C" {

// the library's one error text (errors.h).  The per-header names are aliases of uhc_last_error, kept for the callers of earlier releases
const char *uhc_last_error(void) { return uhc_err().c_str(); }
const char *uhc_nn_last_error(void) { return uhc_last_error(); }
const char *uhc_tc_last_error(void) { return uhc_last_error(); }
const char *uhc_ppo_last_error(void) { return uhc_last_error(); }
const char *uhc_rollout_last_error(void) { return uhc_last_error(); }
const char *uhc_eval_last_error(void) { return uhc_last_error(); }
const char *uhc_track_last_error(void) { return uhc_last_error(); }
const char *uhc_render_last_error(void) { return uhc_last_error(); }
const char *uhc_export_last_error(void) { return uhc_last_error(); }

int uhc_engine_create(const UhcModelHost *model, const UhcEnvCfg *cfg, int num_envs, int device, int precision, UhcEngine **out) {
    if (!model || !cfg || !out || num_envs <= 0 || (precision != 32 && precision != 64)) { uhc_err() = "uhc_engine_create: bad argument"; return -2; }
    CK(cudaSetDevice(device));
    UhcEngine *e = new UhcEngine();
    e->E = num_envs; e->device = device; e->precision = precision; e->launches = 0; e->nshape = model->nshape > 0 ? model->nshape : 1;
    int rc = precision == 32 ? build_view<float>(e, e->evf, model, cfg) : build_view<double>(e, e->evd, model, cfg);
    if (rc) { delete e; return rc; }
    e->base_bf.assign(model->body_f, model->body_f + NB * BODYF); e->base_hull.assign(model->hull, model->hull + (size_t)model->nvert * 3);
    e->base_dof.assign(model->dof_f, model->dof_f + NV * 4);
    e->base_hull_adr.assign(model->hull_adr, model->hull_adr + NB); e->base_hull_num.assign(model->hull_num, model->hull_num + NB);
    e->base_parent.assign(model->parent, model->parent + NB); e->base_sub_end.assign(model->body_sub_end, model->body_sub_end + NB);
    {   // the motion library's FK reads the bone offsets / com positions of every shape variant in fp64, whatever the engine's precision
        std::vector<double> body((size_t)e->nshape * NB * motion::BODY6);
        motion::motion_body_table(model->body_f, BODYF, e->nshape, body.data());
        double *d_body;
        if (dev_copy(e, &d_body, body.data(), body.size())) { delete e; return -1; }
        motion::motion_model_init(e->mo_model, model->parent, model->ee, d_body);
    }
    {   // work-sorted warp slots: opt-in (UHC_SORT_ENVS=1).  At 4096 envs sorting was slower than the identity
        // mapping -- the previous step's iteration total does not predict the per-substep imbalance well enough to pay for itself
        const char *se = getenv("UHC_SORT_ENVS");
        if (se && se[0] == '1' && num_envs > 2 * EPB_F) { CK(cudaMalloc((void **)&e->d_order, (size_t)num_envs * sizeof(int))); e->allocs.push_back(e->d_order); }
    }
    if (precision == 32) {
        CK(cudaFuncSetAttribute(k_env_step<float, EPB_F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<float, EPB_F>()));
        CK(cudaFuncSetAttribute(k_env_step<float, EPB_F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<float, EPB_F>()));
        CK(cudaFuncSetAttribute(k_env_reset<float, EPB_F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<float, EPB_F>()));
        CK(cudaFuncSetAttribute(k_eval_reseat<float, EPB_F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<float, EPB_F>()));
        int resident = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, k_env_step<float, EPB_F>, 32 * EPB_F, step_smem<float, EPB_F>()));
        if (resident < 1) { uhc_err() = "uhc_engine_create: k_env_step<float> with " + std::to_string(EPB_F) + " envs per block does not fit one SM"; delete e; return -3; }
    } else {
        CK(cudaFuncSetAttribute(k_env_step<double, EPB_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<double, EPB_D>()));
        CK(cudaFuncSetAttribute(k_env_step<double, EPB_D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<double, EPB_D>()));
        CK(cudaFuncSetAttribute(k_env_reset<double, EPB_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<double, EPB_D>()));
        CK(cudaFuncSetAttribute(k_eval_reseat<double, EPB_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)step_smem<double, EPB_D>()));
    }
    const size_t E = num_envs;
    CK(cudaMalloc((void **)&e->d_act, E * MAX_ACT_DIM * 4)); CK(cudaMalloc((void **)&e->d_obs, E * (size_t)(precision == 32 ? e->evf.cfg.obs_dim : e->evd.cfg.obs_dim) * 4)); CK(cudaMalloc((void **)&e->d_rew, E * 4));
    CK(cudaMalloc((void **)&e->d_cinfo, E * 5 * 4)); CK(cudaMalloc((void **)&e->d_pct, E * 4)); CK(cudaMalloc((void **)&e->d_fail, E * 4)); CK(cudaMalloc((void **)&e->d_end, E * 4));
    for (void *p : {(void *)e->d_act, (void *)e->d_obs, (void *)e->d_rew, (void *)e->d_cinfo, (void *)e->d_pct, (void *)e->d_fail, (void *)e->d_end}) e->allocs.push_back(p);
    *out = e;
    return 0;
}

void uhc_engine_destroy(UhcEngine *e) {
    if (!e) return;
    cudaSetDevice(e->device);
    for (void *p : e->allocs) cudaFree(p);
    if (e->d_expert) cudaFree(e->d_expert);
    if (e->d_shape) cudaFree(e->d_shape);
    if (e->d_clip_adr) cudaFree(e->d_clip_adr);
    if (e->d_clip_cdf) cudaFree(e->d_clip_cdf);
    if (e->d_clip_model) cudaFree(e->d_clip_model);
    if (e->d_ids) cudaFree(e->d_ids);
    if (e->h_ids) cudaFreeHost(e->h_ids);
    if (e->ids_done) cudaEventDestroy(e->ids_done);
    if (e->d_qv) cudaFree(e->d_qv);
    if (e->d_keep) cudaFree(e->d_keep);
    if (e->d_keep_t) cudaFree(e->d_keep_t);
    if (e->d_gather) cudaFree(e->d_gather);
    if (e->d_gather_i) cudaFree(e->d_gather_i);
    for (void *p : {(void *)e->cur.pct, (void *)e->cur.start, (void *)e->cur.meta, (void *)e->cur.p, (void *)e->cur.cnt, (void *)e->cur.rank, (void *)e->cur.ncl, (void *)e->d_reseed, (void *)e->d_push}) if (p) cudaFree(p);
    if (e->d_slot_hull) cudaFree(e->d_slot_hull);
    subjx::builder_free(e->subj);
    delete e;
}

// cumulative clip sampling weights: explicit weights (uhc_set_clip_weights) or the sample_keys rule of the reference
// (len // t_max + 1 copies per clip, dataset_amass_single.py:138-142)
static int upload_clip_cdf(UhcEngine *e) {
    const int nclips = e->num_clips;
    if (nclips <= 0) return 0;
    const int tmax = e->precision == 32 ? e->evf.cfg.t_max : e->evd.cfg.t_max;
    std::vector<float> cdf(nclips); double acc = 0.0;
    for (int i = 0; i < nclips; i++) {
        acc += e->clip_w.empty() ? (double)(tmax > 0 ? e->clip_len_h[i] / tmax + 1 : 1) : (double)e->clip_w[i];
        cdf[i] = (float)acc;
    }
    if (!e->d_clip_cdf) CK(cudaMalloc((void **)&e->d_clip_cdf, nclips * sizeof(float)));
    CK(cudaMemcpy(e->d_clip_cdf, cdf.data(), nclips * sizeof(float), cudaMemcpyHostToDevice));
    e->evf.clip_cdf = e->d_clip_cdf; e->evd.clip_cdf = e->d_clip_cdf;
    return 0;
}

static int cur_weights(UhcEngine *e);
static void cur_free(UhcEngine *e);
static void cur_view(UhcEngine *e);

int uhc_engine_set_cfg(UhcEngine *e, const UhcEnvCfg *cfg) {
    if (!e || !cfg) { uhc_err() = "uhc_engine_set_cfg: null"; return -2; }
    e->view_gen++;
    CK(cudaSetDevice(e->device));
    const int old_tmax = e->precision == 32 ? e->evf.cfg.t_max : e->evd.cfg.t_max;
    const int old_obs_dim = uhc_engine_obs_dim(e);
    if (e->precision == 32) { fill_cfg(e->evf.cfg, cfg); e->evf.cfg.num_clips = e->num_clips; } else { fill_cfg(e->evd.cfg, cfg); e->evd.cfg.num_clips = e->num_clips; }
    if (uhc_engine_obs_dim(e) != old_obs_dim) { uhc_err() = "uhc_engine_set_cfg: the observation width cannot change on a live engine (buffers are sized at creation)"; return -2; }
    if (cfg->t_max != old_tmax && e->clip_w.empty()) { CK(cudaDeviceSynchronize()); return e->cur.M ? cur_weights(e) : upload_clip_cdf(e); }   // the sample_keys weights depend on t_max
    return 0;
}

// replaces the clip table (shared by uhc_load_clips and uhc_load_motions): clip addresses, sampling CDF back to the sample_keys rule,
// clip models back to variant 0, every env record invalidated, shapes uploaded; d_expert is allocated (uninitialised) for the caller
static int new_clip_table(UhcEngine *e, int nclips, const int *clip_len, const double *shape_host) {
    e->view_gen++; e->table_gen++;
    if (e->cur.M && nclips != e->num_clips) cur_free(e);   // the histories belong to the old clips
    std::vector<int> adr(nclips + 1, 0);
    for (int i = 0; i < nclips; i++) adr[i + 1] = adr[i] + clip_len[i];
    const size_t nf = (size_t)adr[nclips] * EX_SIZE, ns = (size_t)nclips * 17;
    if (e->d_expert) { cudaFree(e->d_expert); cudaFree(e->d_shape); cudaFree(e->d_clip_adr); cudaFree(e->d_clip_cdf); e->d_expert = e->d_shape = nullptr; e->d_clip_adr = nullptr; e->d_clip_cdf = nullptr; }
    CK(cudaMalloc((void **)&e->d_clip_adr, (nclips + 1) * sizeof(int)));
    CK(cudaMemcpy(e->d_clip_adr, adr.data(), (nclips + 1) * sizeof(int), cudaMemcpyHostToDevice));
    e->num_clips = nclips; e->clip_len_h.assign(clip_len, clip_len + nclips); e->clip_adr_h = adr; e->clip_w.clear();
    e->evf.cfg.num_clips = nclips; e->evd.cfg.num_clips = nclips;
    if (upload_clip_cdf(e)) return -1;
    if (e->cur.M) {                                          // same clip count: the curriculum keeps its history and rewrites the new CDF
        if (cur_weights(e)) return -1;
        cur_view(e);                                         // the CDF moved: the rollout's graphs must capture the new one
    }
    if (e->d_clip_model) { cudaFree(e->d_clip_model); e->d_clip_model = nullptr; }
    e->evf.clip_model = nullptr; e->evd.clip_model = nullptr;
    // every env record points into the OLD clip table: invalidate them all (len = 0); the step kernel skips (and flags) an env
    // until uhc_env_reset gives it a slice of the new table
    CK(cudaMemset(e->precision == 32 ? e->evf.istate : e->evd.istate, 0, (size_t)e->E * SI_SIZE * sizeof(int)));
    if (e->precision == 32) {
        std::vector<float> s(ns);
        for (size_t i = 0; i < ns; i++) s[i] = (float)shape_host[i];
        CK(cudaMalloc(&e->d_expert, nf * 4)); CK(cudaMalloc(&e->d_shape, ns * 4));
        CK(cudaMemcpy(e->d_shape, s.data(), ns * 4, cudaMemcpyHostToDevice));
        e->evf.expert = (const float *)e->d_expert; e->evf.clip_shape = (const float *)e->d_shape; e->evf.clip_adr = e->d_clip_adr;
    } else {
        CK(cudaMalloc(&e->d_expert, nf * 8)); CK(cudaMalloc(&e->d_shape, ns * 8));
        CK(cudaMemcpy(e->d_shape, shape_host, ns * 8, cudaMemcpyHostToDevice));
        e->evd.expert = (const double *)e->d_expert; e->evd.clip_shape = (const double *)e->d_shape; e->evd.clip_adr = e->d_clip_adr;
    }
    return 0;
}

int uhc_load_clips(UhcEngine *e, int nclips, const int *clip_len, const double *frames_host, const double *shape_host) {
    if (!e || nclips <= 0 || !clip_len || !frames_host || !shape_host) { uhc_err() = "uhc_load_clips: bad argument"; return -2; }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    size_t nframes = 0;
    for (int i = 0; i < nclips; i++) { if (clip_len[i] < 2) { uhc_err() = "uhc_load_clips: clip shorter than 2 frames"; return -2; } nframes += clip_len[i]; }
    if (new_clip_table(e, nclips, clip_len, shape_host)) return -1;
    const size_t nf = nframes * EX_SIZE;
    if (e->precision == 32) {
        std::vector<float> f(nf);
        for (size_t i = 0; i < nf; i++) f[i] = (float)frames_host[i];
        CK(cudaMemcpy(e->d_expert, f.data(), nf * 4, cudaMemcpyHostToDevice));
    } else {
        CK(cudaMemcpy(e->d_expert, frames_host, nf * 8, cudaMemcpyHostToDevice));
    }
    return 0;
}

// pinned / device staging of uhc_load_motions: two buffers, so the host fills one chunk while the device copies and expands the other
struct MotionStaging {
    double *h[2] = {nullptr, nullptr}, *d[2] = {nullptr, nullptr}; int *d_fk = nullptr;
    cudaEvent_t ev[2][3] = {};   // per buffer: copy start, kernel start, kernel end
    ~MotionStaging() {
        for (int s = 0; s < 2; s++) {
            if (h[s]) cudaFreeHost(h[s]);
            if (d[s]) cudaFree(d[s]);
            for (int k = 0; k < 3; k++) if (ev[s][k]) cudaEventDestroy(ev[s][k]);
        }
        if (d_fk) cudaFree(d_fk);
    }
};
static void add_elapsed(float *acc, cudaEvent_t a, cudaEvent_t b) { float ms = 0.f; if (cudaEventElapsedTime(&ms, a, b) == cudaSuccess) *acc += ms; }

int uhc_load_motions(UhcEngine *e, int nclips, const int *clip_len, int kind, int pose_dim, const double *rows_host, const double *shape_host,
                     const int *fk_model, int chunk_frames) {
    if (!e || nclips <= 0 || !clip_len || !rows_host || !shape_host) { uhc_err() = "uhc_load_motions: bad argument"; return -2; }
    if (kind != UHC_MOTION_SMPL && kind != UHC_MOTION_QPOS) { uhc_err() = "uhc_load_motions: kind must be UHC_MOTION_SMPL or UHC_MOTION_QPOS"; return -2; }
    if (kind == UHC_MOTION_SMPL ? (pose_dim != 72 && pose_dim != 156) : pose_dim != NQ) { uhc_err() = "uhc_load_motions: pose_dim must be 72 or 156 (UHC_MOTION_SMPL) or 76 (UHC_MOTION_QPOS)"; return -2; }
    if (chunk_frames < 0) { uhc_err() = "uhc_load_motions: chunk_frames < 0"; return -2; }
    long long total = 0;
    for (int i = 0; i < nclips; i++) {
        if (clip_len[i] < 2) { uhc_err() = "uhc_load_motions: clip shorter than 2 frames"; return -2; }
        total += clip_len[i];
        if (fk_model && (fk_model[i] < 0 || fk_model[i] >= e->nshape)) { uhc_err() = "uhc_load_motions: fk_model index out of range"; return -2; }
    }
    if (total > 0x7fffffffLL) { uhc_err() = "uhc_load_motions: more than 2^31 - 1 frames"; return -2; }
    const int row_w = kind == UHC_MOTION_SMPL ? pose_dim + 3 : NQ;
    const int cap = chunk_frames > 0 ? chunk_frames : 32768;
    // chunks of whole clips, each of at most `cap` frames unless a single clip is longer
    std::vector<int> cut(1, 0); size_t rows_max = 0;
    {
        long long n = 0;
        for (int i = 0; i < nclips; i++) {
            if (n > 0 && n + clip_len[i] > cap) { cut.push_back(i); rows_max = (size_t)n > rows_max ? (size_t)n : rows_max; n = 0; }
            n += clip_len[i];
        }
        cut.push_back(nclips); rows_max = (size_t)n > rows_max ? (size_t)n : rows_max;
    }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    MotionStaging st;
    const size_t stage_bytes = rows_max * row_w * sizeof(double);
    for (int s = 0; s < 2; s++) {
        CK(cudaHostAlloc((void **)&st.h[s], stage_bytes, cudaHostAllocDefault)); CK(cudaMalloc((void **)&st.d[s], stage_bytes));
        for (int k = 0; k < 3; k++) CK(cudaEventCreate(&st.ev[s][k]));
    }
    if (fk_model) { CK(cudaMalloc((void **)&st.d_fk, nclips * sizeof(int))); CK(cudaMemcpy(st.d_fk, fk_model, nclips * sizeof(int), cudaMemcpyHostToDevice)); }
    if (new_clip_table(e, nclips, clip_len, shape_host)) return -1;
    e->mo_ms[0] = e->mo_ms[1] = 0.f;
    const int nchunk = (int)cut.size() - 1;
    for (int k = 0; k < nchunk; k++) {
        const int s = k & 1, c0 = cut[k], c1 = cut[k + 1];
        const int f0 = e->clip_adr_h[c0], nf = e->clip_adr_h[c1] - f0;
        if (k >= 2) {   // buffer s was last used by chunk k - 2: wait for its kernel, then take its timings
            CK(cudaEventSynchronize(st.ev[s][2]));
            add_elapsed(&e->mo_ms[1], st.ev[s][0], st.ev[s][1]); add_elapsed(&e->mo_ms[0], st.ev[s][1], st.ev[s][2]);
        }
        memcpy(st.h[s], rows_host + (size_t)f0 * row_w, (size_t)nf * row_w * sizeof(double));
        CK(cudaEventRecord(st.ev[s][0], 0));
        CK(cudaMemcpyAsync(st.d[s], st.h[s], (size_t)nf * row_w * sizeof(double), cudaMemcpyHostToDevice, 0));
        CK(cudaEventRecord(st.ev[s][1], 0));
        CK(e->precision == 32 ? motion::launch_motion_frames<float>(e->mo_model, kind, pose_dim, st.d[s], e->d_clip_adr, st.d_fk, c0, c1, nf, (float *)e->d_expert, 0)
                              : motion::launch_motion_frames<double>(e->mo_model, kind, pose_dim, st.d[s], e->d_clip_adr, st.d_fk, c0, c1, nf, (double *)e->d_expert, 0));
        CK(cudaEventRecord(st.ev[s][2], 0));
        e->launches++;
    }
    CK(cudaDeviceSynchronize());
    for (int k = nchunk > 2 ? nchunk - 2 : 0; k < nchunk; k++) {
        const int s = k & 1;
        add_elapsed(&e->mo_ms[1], st.ev[s][0], st.ev[s][1]); add_elapsed(&e->mo_ms[0], st.ev[s][1], st.ev[s][2]);
    }
    return 0;
}

int uhc_get_clip_frames(UhcEngine *e, int clip, int first, int n, double *out_host) {
    if (!e || !out_host || clip < 0 || clip >= e->num_clips || first < 0 || n < 0 || first + n > e->clip_len_h[clip]) { uhc_err() = "uhc_get_clip_frames: bad argument"; return -2; }
    if (!e->d_expert) { uhc_err() = "uhc_get_clip_frames: no clips loaded"; return -3; }
    if (n == 0) return 0;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    const size_t off = ((size_t)e->clip_adr_h[clip] + first) * EX_SIZE, cnt = (size_t)n * EX_SIZE;
    if (e->precision == 32) {
        std::vector<float> f(cnt);
        CK(cudaMemcpy(f.data(), (const float *)e->d_expert + off, cnt * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < cnt; i++) out_host[i] = (double)f[i];
    } else {
        CK(cudaMemcpy(out_host, (const double *)e->d_expert + off, cnt * 8, cudaMemcpyDeviceToHost));
    }
    return 0;
}

int uhc_load_motions_time(const UhcEngine *e, float *out2) {
    if (!e || !out2) { uhc_err() = "uhc_load_motions_time: bad argument"; return -2; }
    out2[0] = e->mo_ms[0]; out2[1] = e->mo_ms[1];
    return 0;
}

int uhc_set_neutral_pose(UhcEngine *e, const double *qpos76, const double *qvel75) {
    if (!e || !qpos76 || !qvel75) { uhc_err() = "uhc_set_neutral_pose: bad argument"; return -2; }
    e->view_gen++;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    std::vector<double> h(NQ + NV);
    memcpy(h.data(), qpos76, NQ * 8); memcpy(h.data() + NQ, qvel75, NV * 8);
    if (e->precision == 32) { const float *d; if (dev_copy_real<float>(e, &d, h.data(), NQ + NV)) return -1; e->evf.neutral = d; }
    else { const double *d; if (dev_copy_real<double>(e, &d, h.data(), NQ + NV)) return -1; e->evd.neutral = d; }
    return 0;
}

int uhc_set_clip_weights(UhcEngine *e, int nclips, const float *weights_host) {
    if (!e || nclips != e->num_clips) { uhc_err() = "uhc_set_clip_weights: call after uhc_load_clips with one weight per clip"; return -2; }
    if (e->cur.M) { uhc_err() = "uhc_set_clip_weights: the device curriculum owns the clip weights (uhc_curriculum_enable with max_freq 0 turns it off)"; return -2; }
    e->view_gen++;
    CK(cudaSetDevice(e->device));
    if (!weights_host) e->clip_w.clear();
    else {
        double tot = 0; for (int i = 0; i < nclips; i++) { if (!(weights_host[i] >= 0.f)) { uhc_err() = "uhc_set_clip_weights: negative / NaN weight"; return -2; } tot += weights_host[i]; }
        if (!(tot > 0)) { uhc_err() = "uhc_set_clip_weights: all weights are zero"; return -2; }
        e->clip_w.assign(weights_host, weights_host + nclips);
    }
    CK(cudaDeviceSynchronize());
    return upload_clip_cdf(e);
}

int uhc_set_clip_models(UhcEngine *e, int nclips, const int *clip_model) {
    if (!e || !clip_model || nclips != e->num_clips) { uhc_err() = "uhc_set_clip_models: call after uhc_load_clips with one entry per clip"; return -2; }
    e->view_gen++;
    for (int i = 0; i < nclips; i++) if (clip_model[i] < 0 || clip_model[i] >= e->nshape) { uhc_err() = "uhc_set_clip_models: shape index out of range"; return -2; }
    CK(cudaSetDevice(e->device));
    if (e->d_clip_model) cudaFree(e->d_clip_model);
    CK(cudaMalloc((void **)&e->d_clip_model, nclips * sizeof(int)));
    CK(cudaMemcpy(e->d_clip_model, clip_model, nclips * sizeof(int), cudaMemcpyHostToDevice));
    e->evf.clip_model = e->d_clip_model; e->evd.clip_model = e->d_clip_model;
    return 0;
}

int uhc_env_reset(UhcEngine *e, int n, const int *env_ids_host, const int *clip_host, const int *start_host, const int *len_host,
                  const float *qpos_dev, const float *qvel_dev, float *obs_dev, void *stream) {
    if (!e || n <= 0 || !env_ids_host || !clip_host || !start_host || !len_host) { uhc_err() = "uhc_env_reset: bad argument"; return -2; }
    if (!e->d_expert) { uhc_err() = "uhc_env_reset: no clips loaded"; return -3; }
    CK(cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n; i++) {
        if (env_ids_host[i] < 0 || env_ids_host[i] >= e->E) { uhc_err() = "uhc_env_reset: env id out of range"; return -2; }
        const int c = clip_host[i];
        if (c < 0 || c >= e->num_clips) { uhc_err() = "uhc_env_reset: clip index out of range"; return -2; }
        if (start_host[i] < 0 || len_host[i] < 1 || start_host[i] + len_host[i] > e->clip_len_h[c]) { uhc_err() = "uhc_env_reset: (start, length) outside the clip"; return -2; }
    }
    // the arguments travel through a pinned staging buffer owned by the engine, so the caller's arrays are free on return and the
    // call stays asynchronous: the only wait is for the PREVIOUS reset's kernel to have consumed the staging buffer
    if (!e->ids_done) CK(cudaEventCreateWithFlags(&e->ids_done, cudaEventDisableTiming));
    else CK(cudaEventSynchronize(e->ids_done));
    if (e->ids_cap < n) {
        if (e->d_ids) cudaFree(e->d_ids);
        if (e->h_ids) cudaFreeHost(e->h_ids);
        const int cap = n > 256 ? n : 256;
        CK(cudaMalloc((void **)&e->d_ids, (size_t)4 * cap * sizeof(int))); CK(cudaHostAlloc((void **)&e->h_ids, (size_t)4 * cap * sizeof(int), cudaHostAllocDefault));
        e->ids_cap = cap;
    }
    memcpy(e->h_ids, env_ids_host, n * sizeof(int)); memcpy(e->h_ids + n, clip_host, n * sizeof(int));
    memcpy(e->h_ids + 2 * n, start_host, n * sizeof(int)); memcpy(e->h_ids + 3 * n, len_host, n * sizeof(int));
    CK(cudaMemcpyAsync(e->d_ids, e->h_ids, (size_t)4 * n * sizeof(int), cudaMemcpyHostToDevice, st));
    if (e->precision == 32)
        k_env_reset<float, EPB_F><<<(n + EPB_F - 1) / EPB_F, 32 * EPB_F, step_smem<float, EPB_F>(), st>>>(e->evf, n, e->d_ids, e->d_ids + n, e->d_ids + 2 * n, e->d_ids + 3 * n, qpos_dev, qvel_dev, obs_dev);
    else
        k_env_reset<double, EPB_D><<<(n + EPB_D - 1) / EPB_D, 32 * EPB_D, step_smem<double, EPB_D>(), st>>>(e->evd, n, e->d_ids, e->d_ids + n, e->d_ids + 2 * n, e->d_ids + 3 * n, qpos_dev, qvel_dev, obs_dev);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e->ids_done, st));
    e->launches++;
    return 0;
}

#ifdef UHC_PHASE_CLOCKS
// Builds with -DUHC_PHASE_CLOCKS only (scripts/step_phase_cycles.py; not part of the library's API): from the next launch on, every warp of
// k_env_step adds the clock64() cycles of each phase of its control step (sim_core.h, PC_*) to buf[env][phase] -- device memory of
// E x NPHASE int64 the caller zeroes; null stops the accounting.  Returns NPHASE.  Graphs captured before this call keep the old view.
int uhc_phase_clocks(UhcEngine *e, long long *buf) {
    if (!e) { uhc_err() = "uhc_phase_clocks: bad argument"; return -2; }
    e->evf.phase_cyc = buf; e->evd.phase_cyc = buf;
    e->view_gen++;
    return NPHASE;
}
#endif

int uhc_env_step(UhcEngine *e, const float *actions_dev, float *obs_dev, float *reward_dev, float *cinfo_dev, int *fail_dev, int *end_dev,
                 float *percent_dev, float *torque_dev, void *stream) {
    if (!e || !actions_dev) { uhc_err() = "uhc_env_step: bad argument"; return -2; }
    if (!e->d_expert) { uhc_err() = "uhc_env_step: no clips loaded"; return -3; }
    CK(cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (e->d_order) { k_order_envs<<<1, 1024, 0, st>>>(e->precision == 32 ? e->evf.istate : e->evd.istate, e->E, e->d_order); e->launches++; }
    const bool cur = e->cur.M > 0;     // the curriculum variant: start log and curriculum sampler
    if (e->precision == 32)
        (cur ? k_env_step<float, EPB_F, true> : k_env_step<float, EPB_F>)<<<(e->E + EPB_F - 1) / EPB_F, 32 * EPB_F, step_smem<float, EPB_F>(), st>>>(e->evf, actions_dev, obs_dev, reward_dev, cinfo_dev, fail_dev, end_dev, percent_dev, torque_dev, e->d_order);
    else
        (cur ? k_env_step<double, EPB_D, true> : k_env_step<double, EPB_D>)<<<(e->E + EPB_D - 1) / EPB_D, 32 * EPB_D, step_smem<double, EPB_D>(), st>>>(e->evd, actions_dev, obs_dev, reward_dev, cinfo_dev, fail_dev, end_dev, percent_dev, torque_dev, e->d_order);
    CK(cudaGetLastError());
    e->launches++;
    return 0;
}

int uhc_env_step_host(UhcEngine *e, const float *actions_host, float *obs_host, float *reward_host, float *cinfo_host, int *fail_host,
                      int *end_host, float *percent_host) {
    if (!e || !actions_host) { uhc_err() = "uhc_env_step_host: bad argument"; return -2; }
    CK(cudaSetDevice(e->device));
    const size_t E = e->E;
    CK(cudaMemcpyAsync(e->d_act, actions_host, E * (size_t)uhc_engine_act_dim(e) * 4, cudaMemcpyHostToDevice, 0));
    int rc = uhc_env_step(e, e->d_act, e->d_obs, e->d_rew, e->d_cinfo, e->d_fail, e->d_end, e->d_pct, nullptr, nullptr);
    if (rc) return rc;
    if (obs_host) CK(cudaMemcpyAsync(obs_host, e->d_obs, E * (size_t)uhc_engine_obs_dim(e) * 4, cudaMemcpyDeviceToHost, 0));
    if (reward_host) CK(cudaMemcpyAsync(reward_host, e->d_rew, E * 4, cudaMemcpyDeviceToHost, 0));
    if (cinfo_host) CK(cudaMemcpyAsync(cinfo_host, e->d_cinfo, E * 5 * 4, cudaMemcpyDeviceToHost, 0));
    if (fail_host) CK(cudaMemcpyAsync(fail_host, e->d_fail, E * 4, cudaMemcpyDeviceToHost, 0));
    if (end_host) CK(cudaMemcpyAsync(end_host, e->d_end, E * 4, cudaMemcpyDeviceToHost, 0));
    if (percent_host) CK(cudaMemcpyAsync(percent_host, e->d_pct, E * 4, cudaMemcpyDeviceToHost, 0));
    CK(cudaStreamSynchronize(0));
    return 0;
}

// state of n envs in one gather kernel + one copy: out = [n][319] doubles (qpos76 qvel75 xpos72 bquat96), iout = [n][8]
int uhc_env_get_state_batch(UhcEngine *e, int n, const int *env_ids_host, double *out_host, int *istate_host) {
    if (!e || n <= 0 || !env_ids_host || !out_host) { uhc_err() = "uhc_env_get_state_batch: bad argument"; return -2; }
    for (int i = 0; i < n; i++) if (env_ids_host[i] < 0 || env_ids_host[i] >= e->E) { uhc_err() = "uhc_env_get_state_batch: env id out of range"; return -2; }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    if (e->gather_cap < n) {
        if (e->d_gather) { cudaFree(e->d_gather); cudaFree(e->d_gather_i); }
        CK(cudaMalloc((void **)&e->d_gather, (size_t)n * 319 * sizeof(double))); CK(cudaMalloc((void **)&e->d_gather_i, (size_t)n * (SI_SIZE + 1) * sizeof(int)));
        e->gather_cap = n;
    }
    int *d_idl = e->d_gather_i + (size_t)n * SI_SIZE;
    CK(cudaMemcpy(d_idl, env_ids_host, n * sizeof(int), cudaMemcpyHostToDevice));
    if (e->precision == 32) k_gather_state<float><<<n, 128>>>(e->evf.state, e->evf.istate, d_idl, n, e->d_gather, e->d_gather_i);
    else k_gather_state<double><<<n, 128>>>(e->evd.state, e->evd.istate, d_idl, n, e->d_gather, e->d_gather_i);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out_host, e->d_gather, (size_t)n * 319 * sizeof(double), cudaMemcpyDeviceToHost));
    if (istate_host) CK(cudaMemcpy(istate_host, e->d_gather_i, (size_t)n * SI_SIZE * sizeof(int), cudaMemcpyDeviceToHost));
    return 0;
}

int uhc_env_get_state(UhcEngine *e, int env, double *qpos76, double *qvel75, double *xpos72, double *bquat96, int *istate8) {
    if (!e || env < 0 || env >= e->E) { uhc_err() = "uhc_env_get_state: bad argument"; return -2; }
    double out[319]; int is[SI_SIZE];
    int rc = uhc_env_get_state_batch(e, 1, &env, out, is);
    if (rc) return rc;
    if (qpos76) memcpy(qpos76, out, NQ * 8);
    if (qvel75) memcpy(qvel75, out + 76, NV * 8);
    if (xpos72) memcpy(xpos72, out + 151, 72 * 8);
    if (bquat96) memcpy(bquat96, out + 223, 96 * 8);
    if (istate8) memcpy(istate8, is, sizeof is);
    return 0;
}

// fail_safe (humanoid_im.py:902-905) for n envs at once: overwrite qpos/qvel, run sim.forward(), keep cur_t and the body quats.
// One reset-with-override launch for all of them; no allocation in the steady state.
int uhc_env_set_state_batch(UhcEngine *e, int n, const int *env_ids_host, const double *qpos_host, const double *qvel_host) {
    if (!e || n <= 0 || !env_ids_host || !qpos_host || !qvel_host) { uhc_err() = "uhc_env_set_state_batch: bad argument"; return -2; }
    for (int i = 0; i < n; i++) if (env_ids_host[i] < 0 || env_ids_host[i] >= e->E) { uhc_err() = "uhc_env_set_state_batch: env id out of range"; return -2; }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    const size_t rs = e->precision == 32 ? 4 : 8;
    if (e->qv_cap < n) {
        if (e->d_qv) { cudaFree(e->d_qv); cudaFree(e->d_keep); cudaFree(e->d_keep_t); }
        CK(cudaMalloc((void **)&e->d_qv, (size_t)n * (NQ + NV) * 4)); CK(cudaMalloc(&e->d_keep, (size_t)n * 192 * 8)); CK(cudaMalloc((void **)&e->d_keep_t, (size_t)n * 2 * sizeof(int)));
        e->qv_cap = n;
    }
    (void)rs;
    std::vector<float> qv((size_t)n * (NQ + NV));
    for (int i = 0; i < n; i++) { for (int k = 0; k < NQ; k++) qv[(size_t)i * NQ + k] = (float)qpos_host[(size_t)i * NQ + k]; for (int k = 0; k < NV; k++) qv[(size_t)n * NQ + (size_t)i * NV + k] = (float)qvel_host[(size_t)i * NV + k]; }
    CK(cudaMemcpy(e->d_qv, qv.data(), qv.size() * 4, cudaMemcpyHostToDevice));
    std::vector<int> is((size_t)n * SI_SIZE), clip(n), start(n), len(n);
    std::vector<double> tmp((size_t)n * 319);
    int rc = uhc_env_get_state_batch(e, n, env_ids_host, tmp.data(), is.data());
    if (rc) return rc;
    for (int i = 0; i < n; i++) {
        clip[i] = is[(size_t)i * SI_SIZE + SI_CLIP]; start[i] = is[(size_t)i * SI_SIZE + SI_START]; len[i] = is[(size_t)i * SI_SIZE + SI_LEN];
        if (len[i] < 2 || clip[i] < 0 || clip[i] >= e->num_clips) { uhc_err() = "uhc_env_set_state_batch: env has no valid episode (reset it first)"; return -2; }
    }
    int *d_idl = e->d_keep_t + n;
    CK(cudaMemcpy(d_idl, env_ids_host, n * sizeof(int), cudaMemcpyHostToDevice));
    if (e->precision == 32) k_save_restore_bquat<float><<<n, 64>>>(e->evf.state, e->evf.istate, d_idl, n, (float *)e->d_keep, e->d_keep_t, 0);
    else k_save_restore_bquat<double><<<n, 64>>>(e->evd.state, e->evd.istate, d_idl, n, (double *)e->d_keep, e->d_keep_t, 0);
    rc = uhc_env_reset(e, n, env_ids_host, clip.data(), start.data(), len.data(), e->d_qv, e->d_qv + (size_t)n * NQ, nullptr, nullptr);
    if (rc) return rc;
    if (e->precision == 32) k_save_restore_bquat<float><<<n, 64>>>(e->evf.state, e->evf.istate, d_idl, n, (float *)e->d_keep, e->d_keep_t, 1);
    else k_save_restore_bquat<double><<<n, 64>>>(e->evd.state, e->evd.istate, d_idl, n, (double *)e->d_keep, e->d_keep_t, 1);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    return 0;
}

int uhc_env_set_state(UhcEngine *e, int env, const double *qpos76, const double *qvel75) {
    return uhc_env_set_state_batch(e, 1, &env, qpos76, qvel75);
}

// device counters: out[0] = env-steps failed because a body's contacts did not fit the work set (MAXCON), out[1] = env-steps
// skipped on an invalid (stale / never reset) env record
int uhc_engine_counters(UhcEngine *e, int *out4) {
    if (!e || !out4) { uhc_err() = "uhc_engine_counters: bad argument"; return -2; }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out4, e->precision == 32 ? e->evf.counters : e->evd.counters, 4 * sizeof(int), cudaMemcpyDeviceToHost));
    return 0;
}

const int *uhc_episode_log_dev(const UhcEngine *e) { return e ? (e->precision == 32 ? e->evf.ep_log : e->evd.ep_log) : nullptr; }
int uhc_num_envs(const UhcEngine *e) { return e ? e->E : -1; }
int uhc_engine_obs_dim(const UhcEngine *e) { return e ? (e->precision == 32 ? e->evf.cfg.obs_dim : e->evd.cfg.obs_dim) : -1; }
int uhc_engine_act_dim(const UhcEngine *e) { return e ? (e->precision == 32 ? e->evf.cfg.act_dim : e->evd.cfg.act_dim) : -1; }
int uhc_kernel_launches(const UhcEngine *e) { return e ? e->launches : -1; }

// ---- device curriculum (include/uhc_rollout.h; kernels in curriculum.cu)
static void cur_view(UhcEngine *e) {   // what the sampler reads: rings, fit_clip, prec_freq
    CurView v;
    v.pct = e->cur.pct; v.start = e->cur.start; v.meta = e->cur.meta; v.max_freq = e->cur.M;
    v.fit_clip = e->cur.M ? e->fit_clip : -1; v.prec_freq = e->cur.M ? e->prec_freq : 0.f;
    e->evf.cur = v; e->evd.cur = v;
    e->view_gen++; e->cur_gen++;
}
static void cur_free(UhcEngine *e) {
    cudaDeviceSynchronize();
    for (void *p : {(void *)e->cur.pct, (void *)e->cur.start, (void *)e->cur.meta, (void *)e->cur.p, (void *)e->cur.cnt, (void *)e->cur.rank, (void *)e->cur.ncl}) if (p) cudaFree(p);
    if (e->d_push) cudaFree(e->d_push);
    e->d_push = nullptr; e->push_cap = 0;
    e->cur = cur::Dev{}; e->cur_cnt_cap = e->cur_rank_cap = 0; e->fit_clip = -1; e->prec_freq = 0.f;
    // the start log is written by the curriculum's step kernel only: back to "never recorded", as on an engine that never enabled it
    int *sl = e->precision == 32 ? e->evf.ep_start_log : e->evd.ep_start_log;
    cudaMemset(sl, 0xFF, (size_t)e->E * sizeof(int));
    cur_view(e);
}
static void cur_bind(UhcEngine *e) {   // the parts of the device state that follow the clip table and the cfg
    e->cur.C = e->num_clips; e->cur.cdf = e->d_clip_cdf; e->cur.clip_adr = e->d_clip_adr;
    e->cur.t_max = e->precision == 32 ? e->evf.cfg.t_max : e->evd.cfg.t_max;
}
static int cur_weights(UhcEngine *e) {  // CDF from the rings as they are, rewritten in place; synchronous (host-side calls only)
    cur_bind(e);
    CK(cur::launch_weights(e->cur, 0));
    CK(cudaDeviceSynchronize());
    return 0;
}
static int cur_scratch(UhcEngine *e, size_t N) {   // the update's count table and rank array for an N-entry log
    const size_t ncnt = (N + cur::UPD_CHUNK - 1) / cur::UPD_CHUNK * (size_t)e->num_clips;
    if (e->cur_cnt_cap < ncnt) { if (e->cur.cnt) cudaFree(e->cur.cnt); e->cur.cnt = nullptr; CK(cudaMalloc((void **)&e->cur.cnt, ncnt * sizeof(int))); e->cur_cnt_cap = ncnt; }
    if (e->cur_rank_cap < N) { if (e->cur.rank) cudaFree(e->cur.rank); e->cur.rank = nullptr; CK(cudaMalloc((void **)&e->cur.rank, N * sizeof(int))); e->cur_rank_cap = N; }
    return 0;
}
static bool cur_check(UhcEngine *e, const char *who) {
    if (!e) { uhc_err() = std::string(who) + ": null engine"; return false; }
    if (!e->cur.M) { uhc_err() = std::string(who) + ": the device curriculum is not enabled"; return false; }
    return true;
}

int uhc_curriculum_enable(UhcEngine *e, int max_freq, double temp, double freq, double prec_freq, int fit_clip) {
    if (!e || max_freq < 0 || max_freq > cur::MAX_FREQ_CAP) { uhc_err() = "uhc_curriculum_enable: max_freq must be 0 .. 4096"; return -2; }
    CK(cudaSetDevice(e->device));
    if (max_freq == 0) {
        if (e->cur.M) { cur_free(e); CK(cudaDeviceSynchronize()); if (upload_clip_cdf(e)) return -1; }
        return 0;
    }
    if (!e->d_expert || e->num_clips <= 0) { uhc_err() = "uhc_curriculum_enable: no clips loaded"; return -2; }
    if (!(temp > 0.0) || !(temp < 1e300)) { uhc_err() = "uhc_curriculum_enable: temp must be a positive number"; return -2; }
    if (!(freq >= 0.0 && freq <= 1.0) || !(prec_freq >= 0.0 && prec_freq <= 1.0)) { uhc_err() = "uhc_curriculum_enable: freq and prec_freq must lie in [0, 1]"; return -2; }
    if (fit_clip < -1 || fit_clip >= e->num_clips) { uhc_err() = "uhc_curriculum_enable: fit_clip must be -1 or a clip index"; return -2; }
    if (e->cur.M != max_freq) {
        if (e->cur.M) cur_free(e);
        const size_t C = e->num_clips, n = C * max_freq;
        CK(cudaMalloc((void **)&e->cur.pct, n * sizeof(float))); CK(cudaMalloc((void **)&e->cur.start, n * sizeof(int)));
        CK(cudaMalloc((void **)&e->cur.meta, 2 * C * sizeof(int))); CK(cudaMalloc((void **)&e->cur.p, C * sizeof(double)));
        CK(cudaMalloc((void **)&e->cur.ncl, C * sizeof(int)));
        CK(cudaMemset(e->cur.pct, 0, n * sizeof(float))); CK(cudaMemset(e->cur.start, 0, n * sizeof(int))); CK(cudaMemset(e->cur.meta, 0, 2 * C * sizeof(int)));
        e->cur.M = max_freq;
    }
    e->cur.temp = temp; e->cur.freq = freq; e->prec_freq = (float)prec_freq; e->fit_clip = fit_clip;
    e->clip_w.clear();
    CK(cudaDeviceSynchronize());
    if (cur_weights(e)) return -1;
    cur_view(e);                         // new rings / fit_clip / prec_freq: the rollout's graphs capture them
    return 0;
}

int uhc_get_clip_cdf(UhcEngine *e, float *out_host) {
    if (!e || !out_host || !e->d_clip_cdf) { uhc_err() = "uhc_get_clip_cdf: bad argument or no clips loaded"; return -2; }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out_host, e->d_clip_cdf, e->num_clips * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}

int uhc_curriculum_update(UhcEngine *e, const UhcRolloutBuf *buf, int T, void *stream) {
    if (!cur_check(e, "uhc_curriculum_update")) return -2;
    if (!buf || !buf->ep_clip || !buf->ep_pct || !buf->ep_start || T <= 0 || T > buf->T_cap) { uhc_err() = "uhc_curriculum_update: needs ep_clip, ep_pct and ep_start rows and 0 < T <= T_cap"; return -2; }
    CK(cudaSetDevice(e->device));
    const size_t N = (size_t)T * e->E;
    if (N > 0x7fffffffu) { uhc_err() = "uhc_curriculum_update: log too long"; return -2; }
    if (cur_scratch(e, N)) return -1;
    cur_bind(e);
    CK(cur::launch_update(e->cur, buf->ep_clip, buf->ep_pct, buf->ep_start, (int)N, (cudaStream_t)stream));
    e->launches += 4;
    return 0;
}

static int cur_to_host(UhcEngine *e, std::vector<int> &meta, std::vector<float> &pct, std::vector<int> &st) {
    const size_t C = e->num_clips, n = C * e->cur.M;
    meta.resize(2 * C); pct.resize(n); st.resize(n);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(meta.data(), e->cur.meta, 2 * C * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(pct.data(), e->cur.pct, n * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(st.data(), e->cur.start, n * sizeof(int), cudaMemcpyDeviceToHost));
    return 0;
}
static int cur_from_host(UhcEngine *e, const std::vector<int> &meta, const std::vector<float> &pct, const std::vector<int> &st) {
    CK(cudaMemcpy(e->cur.meta, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(e->cur.pct, pct.data(), pct.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(e->cur.start, st.data(), st.size() * sizeof(int), cudaMemcpyHostToDevice));
    return cur_weights(e);
}

int uhc_curriculum_push(UhcEngine *e, int n, const int *clip, const float *pct, const int *start) {
    if (!cur_check(e, "uhc_curriculum_push")) return -2;
    if (n < 0 || (n > 0 && (!clip || !pct || !start))) { uhc_err() = "uhc_curriculum_push: bad argument"; return -2; }
    for (int i = 0; i < n; i++) if (clip[i] < 0 || clip[i] >= e->num_clips || start[i] < 0 || !(pct[i] == pct[i])) { uhc_err() = "uhc_curriculum_push: clip out of range, negative start or NaN percent"; return -2; }
    if (n == 0) return 0;
    CK(cudaSetDevice(e->device));
    // the n outcomes are a log of their own: the update's kernels append them in order and rewrite the CDF (one copy, one synchronise)
    if (e->push_cap < n) {
        if (e->d_push) cudaFree(e->d_push);
        e->d_push = nullptr; e->push_cap = 0;
        CK(cudaMalloc((void **)&e->d_push, (size_t)3 * n * sizeof(int))); e->push_cap = n;
    }
    std::vector<int> h((size_t)3 * n);
    memcpy(h.data(), clip, n * sizeof(int)); memcpy(h.data() + n, pct, n * sizeof(float)); memcpy(h.data() + 2 * (size_t)n, start, n * sizeof(int));
    if (cur_scratch(e, n)) return -1;
    CK(cudaMemcpy(e->d_push, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice));
    cur_bind(e);
    CK(cur::launch_update(e->cur, e->d_push, (const float *)(e->d_push + n), e->d_push + 2 * (size_t)n, n, 0));
    CK(cudaStreamSynchronize(0));
    e->launches += 4;
    return 0;
}

int uhc_curriculum_get(UhcEngine *e, int *len_host, float *pct_host, int *start_host) {
    if (!cur_check(e, "uhc_curriculum_get")) return -2;
    if (!len_host || !pct_host || !start_host) { uhc_err() = "uhc_curriculum_get: bad argument"; return -2; }
    CK(cudaSetDevice(e->device));
    std::vector<int> meta, st; std::vector<float> pc;
    if (cur_to_host(e, meta, pc, st)) return -1;
    const int M = e->cur.M;
    for (int c = 0; c < e->num_clips; c++) {
        len_host[c] = meta[2 * c + 1];
        for (int k = 0; k < M; k++) {
            const bool v = k < meta[2 * c + 1];
            const int s = cur::ring_slot(meta.data(), M, c, k);
            pct_host[(size_t)c * M + k] = v ? pc[(size_t)c * M + s] : 0.f; start_host[(size_t)c * M + k] = v ? st[(size_t)c * M + s] : 0;
        }
    }
    return 0;
}

int uhc_curriculum_set(UhcEngine *e, const int *len_host, const float *pct_host, const int *start_host) {
    if (!cur_check(e, "uhc_curriculum_set")) return -2;
    if (!len_host || !pct_host || !start_host) { uhc_err() = "uhc_curriculum_set: bad argument"; return -2; }
    const int M = e->cur.M, C = e->num_clips;
    std::vector<int> meta(2 * (size_t)C), st((size_t)C * M, 0); std::vector<float> pc((size_t)C * M, 0.f);
    for (int c = 0; c < C; c++) {
        if (len_host[c] < 0 || len_host[c] > M) { uhc_err() = "uhc_curriculum_set: history length outside 0 .. max_freq"; return -2; }
        for (int k = 0; k < len_host[c]; k++) {
            const float p = pct_host[(size_t)c * M + k]; const int s = start_host[(size_t)c * M + k];
            if (s < 0 || !(p == p)) { uhc_err() = "uhc_curriculum_set: negative start or NaN percent"; return -2; }
            pc[(size_t)c * M + k] = p; st[(size_t)c * M + k] = s;
        }
        meta[2 * c] = len_host[c] % M; meta[2 * c + 1] = len_host[c];
    }
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    return cur_from_host(e, meta, pc, st);
}

int uhc_curriculum_reseed(UhcEngine *e, float *obs_dev, void *stream) {
    if (!e) { uhc_err() = "uhc_curriculum_reseed: null engine"; return -2; }
    if (!e->d_expert) { uhc_err() = "uhc_curriculum_reseed: no clips loaded"; return -3; }
    CK(cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (!e->d_reseed) CK(cudaMalloc((void **)&e->d_reseed, (size_t)4 * e->E * sizeof(int)));
    const int E = e->E, *r = e->d_reseed;
    if (e->precision == 32) {
        k_cur_sample<float><<<(E + 127) / 128, 128, 0, st>>>(e->evf, e->d_reseed);
        k_env_reset<float, EPB_F><<<(E + EPB_F - 1) / EPB_F, 32 * EPB_F, step_smem<float, EPB_F>(), st>>>(e->evf, E, r, r + E, r + 2 * E, r + 3 * E, nullptr, nullptr, obs_dev);
    } else {
        k_cur_sample<double><<<(E + 127) / 128, 128, 0, st>>>(e->evd, e->d_reseed);
        k_env_reset<double, EPB_D><<<(E + EPB_D - 1) / EPB_D, 32 * EPB_D, step_smem<double, EPB_D>(), st>>>(e->evd, E, r, r + E, r + 2 * E, r + 3 * E, nullptr, nullptr, obs_dev);
    }
    CK(cudaGetLastError());
    e->launches += 2;
    return 0;
}

}  // extern "C"

// ---- the device evaluation's view of the engine (eval_glue.h)
namespace uhc {
namespace evalx {

void engine_refs(UhcEngine *e, EngineRefs *r) {
    const bool f32 = e->precision == 32;
    r->E = e->E; r->precision = e->precision; r->obs_dim = uhc_engine_obs_dim(e); r->act_dim = uhc_engine_act_dim(e); r->num_clips = e->d_expert ? e->num_clips : 0;
    r->state = f32 ? (void *)e->evf.state : (void *)e->evd.state; r->istate = f32 ? e->evf.istate : e->evd.istate;
    r->expert = e->d_expert; r->clip_adr = e->d_clip_adr; r->clip_len_h = e->clip_len_h.data(); r->view_gen = e->view_gen;
    r->obs = e->d_obs; r->act = e->d_act; r->rew = e->d_rew; r->cinfo = e->d_cinfo; r->pct = e->d_pct; r->fail = e->d_fail; r->end = e->d_end;
}

unsigned long long curriculum_gen(const UhcEngine *e) { return e->cur_gen; }

cudaError_t launch_reseat(UhcEngine *e, int n, const int *reseat, cudaStream_t st) {
    if (e->precision == 32) k_eval_reseat<float, EPB_F><<<(n + EPB_F - 1) / EPB_F, 32 * EPB_F, step_smem<float, EPB_F>(), st>>>(e->evf, n, reseat);
    else k_eval_reseat<double, EPB_D><<<(n + EPB_D - 1) / EPB_D, 32 * EPB_D, step_smem<double, EPB_D>(), st>>>(e->evd, n, reseat);
    e->launches++;
    return cudaGetLastError();
}

}  // namespace evalx

// ---- the tracker's view of the engine (track_glue.h)
namespace trackx {

const char *cfg_error(const UhcEngine *e, int H) {
    const bool f32 = e->precision == 32;
    const int obs_v = f32 ? e->evf.cfg.obs_v : e->evd.cfg.obs_v, term = f32 ? e->evf.cfg.term_body : e->evd.cfg.term_body;
    const int ar = f32 ? e->evf.cfg.auto_reset : e->evd.cfg.auto_reset, rv = f32 ? e->evf.cfg.reactive_v : e->evd.cfg.reactive_v;
    const int trail = f32 ? e->evf.cfg.trail_steps : e->evd.cfg.trail_steps, eplen = f32 ? e->evf.cfg.env_episode_len : e->evd.cfg.env_episode_len;
    if (H < 3) return "the window must hold at least 3 rows";
    if (obs_v == 3) return "obs_v 3 reads future frames a stream does not have";
    if (term != 0) return "term_body root / Head read the whole episode window";
    if (ar) return "auto_reset re-seeds episodes from the clip table";
    if (rv == 1) return "reactive_v 1 starts episodes from the neutral pose";
    if (trail < 1 || eplen < H) return "`end` could fire inside the window: needs trail_steps >= 1 and env_episode_len >= window (the caller owns the episode length)";
    return nullptr;
}

int install_table(UhcEngine *e, int H, const int *fk_model, const double *shape) {
    const int E = e->E;
    if (cudaSetDevice(e->device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) { uhc_err() = "cudaDeviceSynchronize failed"; return -1; }
    std::vector<int> lens(E, H);
    std::vector<double> shp;
    if (!shape) { shp.assign((size_t)E * 17, 0.0); shape = shp.data(); }
    if (new_clip_table(e, E, lens.data(), shape)) return -1;
    if (fk_model && uhc_set_clip_models(e, E, fk_model)) return -1;
    if (!fk_model && e->nslot) {                // uhc_track_set_subjects points single envs at their slots
        const std::vector<int> zero(E, 0);
        if (uhc_set_clip_models(e, E, zero.data())) return -1;
    }
    const size_t rs = e->precision == 32 ? 4 : 8;
    cudaError_t ce = cudaMemset(e->d_expert, 0, (size_t)E * H * EX_SIZE * rs);
    if (ce == cudaSuccess)
        ce = e->precision == 32 ? cudaFuncSetAttribute(k_track_obs<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(EPB_OBS * sizeof(Work<float>)))
                                : cudaFuncSetAttribute(k_track_obs<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(EPB_OBS * sizeof(Work<double>)));
    if (ce != cudaSuccess) { uhc_err() = std::string("install_table: ") + cudaGetErrorString(ce); return -1; }
    return 0;
}

unsigned long long table_gen(const UhcEngine *e) { return e->table_gen; }
int num_shapes(const UhcEngine *e) { return e->nshape; }
const motion::MotionModel &motion_model(const UhcEngine *e) { return e->mo_model; }
const int *clip_models(const UhcEngine *e) { return e->d_clip_model; }

UhcModelHost base_model(const UhcEngine *e) {
    UhcModelHost m;
    memset(&m, 0, sizeof m);
    m.body_f = e->base_bf.data(); m.hull = e->base_hull.data(); m.dof_f = e->base_dof.data(); m.nvert = (int)(e->base_hull.size() / 3);
    m.hull_adr = e->base_hull_adr.data(); m.hull_num = e->base_hull_num.data(); m.parent = e->base_parent.data(); m.body_sub_end = e->base_sub_end.data();
    m.nshape = 1;
    return m;
}

// rows first .. first + n - 1 of a table of `row`-wide rows become copies of row 0
template <class T>
__global__ void k_repeat_row(T *__restrict__ t, size_t row, size_t first, int n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)n * row; i += (size_t)gridDim.x * blockDim.x) t[first * row + i] = t[i % row];
}

// *tab (an engine allocation of nold rows) -> a new allocation of nold + extra rows, the extra ones copies of row 0; the old one is freed
template <class T>
static int grow_table(UhcEngine *e, const T **tab, size_t row, int nold, int extra) {
    T *d = nullptr;
    CK(cudaMalloc((void **)&d, row * (nold + extra) * sizeof(T)));
    e->allocs.push_back(d);
    CK(cudaMemcpy(d, *tab, row * nold * sizeof(T), cudaMemcpyDeviceToDevice));
    k_repeat_row<T><<<1024, 256>>>(d, row, nold, extra);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    for (size_t i = 0; i < e->allocs.size(); i++)
        if (e->allocs[i] == (const void *)*tab) { cudaFree(e->allocs[i]); e->allocs.erase(e->allocs.begin() + i); break; }
    *tab = d;
    return 0;
}

template <class Real>
static int grow_model(UhcEngine *e, Model<Real> &M) {
    if (grow_table<Real>(e, &M.body_f, NB * BODYF, e->nshape, e->E) || grow_table<Real>(e, &M.hull, (size_t)M.nvert * 3, e->nshape, e->E)) return -1;
    M.nshape = e->nshape + e->E;
    return 0;
}

int enable_subjects(UhcEngine *e, subjx::Builder *b) {
    subjx::builder_free(e->subj);
    e->subj = b;
    if (e->nslot) return 0;                     // the slots exist: only the basis changes
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());
    e->view_gen++;                              // the tables move: no graph may replay the old pointers
    evalx::drop_rollout_graphs(e);
    if (e->precision == 32 ? grow_model<float>(e, e->evf.model) : grow_model<double>(e, e->evd.model)) return -1;
    const double *body = e->mo_model.body;
    if (grow_table<double>(e, &body, NB * motion::BODY6, e->nshape, e->E)) return -1;
    e->mo_model.body = body;
    const size_t hv = e->base_hull.size();
    CK(cudaMalloc((void **)&e->d_slot_hull, hv * e->E * sizeof(double)));
    CK(cudaMemcpy(e->d_slot_hull, e->base_hull.data(), hv * sizeof(double), cudaMemcpyHostToDevice));
    k_repeat_row<double><<<1024, 256>>>(e->d_slot_hull, hv, 1, e->E - 1);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    e->nslot = e->E;
    return 0;
}

const subjx::Builder *subject_builder(const UhcEngine *e) { return e->nslot ? e->subj : nullptr; }

void slots(UhcEngine *e, Slots *s) {
    const bool f32 = e->precision == 32;
    s->nshape = e->nshape; s->nvert = f32 ? e->evf.model.nvert : e->evd.model.nvert; s->precision = e->precision;
    s->body_f = f32 ? (void *)e->evf.model.body_f : (void *)e->evd.model.body_f;
    s->hull = f32 ? (void *)e->evf.model.hull : (void *)e->evd.model.hull;
    s->body6 = const_cast<double *>(e->mo_model.body); s->hull64 = e->d_slot_hull;
    s->clip_model = e->d_clip_model; s->shape = e->d_shape; s->istate = f32 ? e->evf.istate : e->evd.istate;
}

const double *slot_hulls(const UhcEngine *e) { return e->d_slot_hull; }

cudaError_t launch_obs(UhcEngine *e, float *obs, cudaStream_t st) {
    const int E = e->E;
    if (e->precision == 32) k_track_obs<float><<<(E + EPB_OBS - 1) / EPB_OBS, 32 * EPB_OBS, EPB_OBS * sizeof(Work<float>), st>>>(e->evf, obs);
    else k_track_obs<double><<<(E + EPB_OBS - 1) / EPB_OBS, 32 * EPB_OBS, EPB_OBS * sizeof(Work<double>), st>>>(e->evd, obs);
    e->launches++;
    return cudaGetLastError();
}

}  // namespace trackx
}  // namespace uhc
