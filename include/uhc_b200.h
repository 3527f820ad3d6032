/* uhc_b200.h -- C ABI of the batched (H100) humanoid-imitation engine (libuhc_b200.so).
 *
 * The reference (ZhengyiLuo/UHC) exposes NO native interface: its boundary is duck-typed Python over mujoco-py.
 * Each entry point below names the reference Python call it replaces (file:line under the reference tree); the
 * ctypes binding a maintainer adds on the reference side is shown in INTEGRATION.md and implemented in
 * uhc_b200/engine.py.  All functions return 0 on success, <0 on error (uhc_last_error() gives the text); nothing
 * throws across the ABI.  A per-env solver/NaN failure is not an error: it sets that env's `fail` flag
 * (mirrors the try/except at uhc/envs/humanoid_im.py:1207-1211).
 * Pointers suffixed _dev are CUDA device pointers owned by the caller (e.g. torch tensors); _host are host pointers.
 * One engine per GPU; calls are stream-ordered on the cudaStream_t passed as `stream`; an engine is not thread-safe.
 */
#ifndef UHC_B200_H
#define UHC_B200_H
#ifdef __cplusplus
extern "C" {
#endif

#define UHC_NB 24
#define UHC_NQ 76
#define UHC_NV 75
#define UHC_NU 69
#define UHC_OBS_DIM 657
#define UHC_ACT_DIM 105       /* action width of the default configuration (implicit residual force + meta-PD) */
#define UHC_MAX_ACT_DIM 315   /* explicit residual force + meta-PD */
#define UHC_OBS_DIM_V1 784    /* obs_v 1 (get_full_obs_v1); obs_v 3 is UHC_OBS_DIM * fut_frames */
#define UHC_EX_SIZE 576       /* expert frame record: qpos76 qvel75 wbpos72 wbquat96 bquat96 bangvel72 ee_wpos15 body_com72 (com = its first 3) pad2 */
#define UHC_BODYF 20

typedef struct UhcEngine UhcEngine;

/* Flat humanoid model tables (built by uhc_b200/model.py from the compiled XML+STL model). Replaces the MuJoCo model
 * object created by mujoco_py.load_model_from_xml at uhc/envs/humanoid_im.py:174 / mujoco_env.py:18. */
typedef struct {
    int nvert, nnbr;
    const double *body_f;   /* [24][20] offset3 ipos3 mass inertia6 invweight bsphere4 diffw pad */
    const double *dof_f;    /* [75][4]  armature kp kd torque_limit */
    const double *hull;     /* [nvert][3] convex-hull vertices, body frame */
    const int *hull_adr, *hull_num, *nbr, *nbradr;
    const int *parent, *depth, *child_adr, *child, *body_sub_end;   /* kinematic tree, bodies numbered depth-first */
    const int *ee;          /* [5] end-effector bodies of the reward (smpl_parser.py:228) */
    const int *lvl_tab;     /* [9][5][5] elimination tree of the joint-space solve, hung from the tree's centre body (7 levels for SMPL): per level
                               and lane group: body, parent's group, groups of up to 3 children (-1 none) */
    const int *lvl_pack;    /* [9][5] the same, packed: (body+1) | pgrp<<6 | (cg0+1)<<9 | (cg1+1)<<12 | (cg2+1)<<15 | max children on the level<<18
                               | (first dof of the connecting joint / 3)<<20 | joint crossed backwards<<25 | number of levels<<26 */
    double dt, margin, mu, solref[2], solimp[5], gravz;
    int nshape;             /* number of body-shape variants: body_f = [nshape][24][20], hull = [nshape][nvert][3] (same topology / hull graph) */
    const double *dof_lim;  /* [75][4] joint limits: lower, upper (rad; the xml's default is limited="true"), dof_invweight0, pad.  NULL = no limits */
} UhcModelHost;

/* Task configuration: the cfg attributes HumanoidEnv / world_rfc_implicit_reward read
 * (uhc/envs/humanoid_im.py:85-89,1138-1142,1228-1235; uhc/losses/reward_function.py:14-30). */
typedef struct {
    double base_rot[4], rfc_scale, rfc_lim, rfc_rate, body_diff_thresh;
    int meta_pd, env_episode_len, trail_steps, newton_max_iter;
    double w[5], k[5], newton_tol;
    /* in-kernel re-seeding of finished episodes (agent_copycat.py:503-512 + dataset_amass_single.py:172-253): when auto_reset != 0,
     * an env whose step ends its episode samples a new (clip, start) slice and is reset inside uhc_env_step; obs = reset obs. */
    int auto_reset, t_min, t_max;
    int reactive_v;         /* cfg.reactive_v (copycat_config.py:97): 1 = train-mode episodes start from the standing-neutral pose with probability reactive_rate */
    unsigned long long reset_seed;
    double reactive_rate;   /* cfg.reactive_rate (copycat_config.py:99, default 0.3) */
    /* cfg.residual_force_mode (copycat_config.py:105-109, humanoid_im.py:231-243): 0 = "implicit" (root wrench, 6 action dims),
     * 1 = "explicit" (contact point + force + torque per body through mj_applyFT, 9 x 24 action dims; reward world_rfc_explicit),
     * 2 = cfg.residual_force false (no residual-force dims in the action, nothing applied, the reward's residual-force term is 0).
     * The action row is [69 joint targets | residual-force dims | 30 meta-PD scales when meta_pd]: uhc_engine_act_dim() gives its width. */
    int rfc_mode;
    int vf_slot[UHC_NB];    /* explicit mode: residual-force slot of body b (the reference orders the slots by SMPL_BONE_ORDER_NAMES, smpl_parser.py:11-36) */
    int obs_v;              /* cfg.obs_v (copycat_config.py:88): 2 = get_full_obs_v2 (657 dims, humanoid_im.py:419-503), 1 = get_full_obs_v1 (784 dims, :323-417);
                             * 3 = get_full_obs_v3 (:505-513): fut_frames v2 blocks against the expert frames cur_t + 1 + i * fut_skip (657 * fut_frames dims);
                             * 5 = get_full_obs_v5 (:505-594, 636 + 17 dims), 6 = get_full_obs_v6 (:596-666, 384 + 17 dims; the 17 shape dims only without no_shape);
                             * 0 is read as 2.  uhc_engine_obs_dim() gives the row width of every obs buffer. */
    int fut_frames, fut_skip;   /* cfg.fut_frames / cfg.skip of obs_v 3 (both default to 10 when <= 0, as cc_cfg.get does) */
    int no_shape;               /* != 0: cfg.has_shape false -- the v2 block carries no shape vector (640 dims instead of 657, humanoid_im.py:499-500) */
    /* cfg.env_term_body (humanoid_im.py:1223-1229): 0 = "body" (mean body-position error above body_diff_thresh), 1 = "root" (root height more than 0.1 m below the
     * lowest of the episode's window of the clip, expert["height_lb"]), 2 = "Head" (height of body head_body below expert["head_height_lb"] - 0.1).  The kernel
     * takes the minimum over the window [start, start + len) itself: the reference's expert IS that slice (dataset_amass_single.py:238-244, tools.py:94-95). */
    int term_body, head_body;
    int reward_mul;             /* != 0: reward_id world_rfc_implicit_v1_mul (reward_function.py:174-250): pose * vel * ee * com * (vf if w[4] != 0), same five c_info terms */
} UhcEnvCfg;

const char *uhc_last_error(void);

/* precision: 32 (product) or 64 (fp64 debug build of the same kernels). */
int uhc_engine_create(const UhcModelHost *model, const UhcEnvCfg *cfg, int num_envs, int device, int precision, UhcEngine **out);
void uhc_engine_destroy(UhcEngine *e);
int uhc_engine_set_cfg(UhcEngine *e, const UhcEnvCfg *cfg);

/* Expert tables for C clips (replaces HumanoidEnv.load_expert's per-episode recompute, humanoid_im.py:182-215):
 * frames_host = concatenated [sum(len)][UHC_EX_SIZE] doubles, shape_host = [C][17] (beta16, gender). */
int uhc_load_clips(UhcEngine *e, int nclips, const int *clip_len, const double *frames_host, const double *shape_host);
/* Expert tables built on the device from raw motion (the opt-in alternative to building them on the host with
 * uhc_b200/motion_lib.py and calling uhc_load_clips; same table, same contract).  rows_host = concatenated [sum(len)][row width]
 * doubles of one kind:
 *   UHC_MOTION_SMPL  pose_aa (pose_dim = 72, or 156 for SMPL-H: columns 66:72 are read as zero) then trans (3): smpl_to_qpose
 *                    (smpl_mujoco.py:543-607) then qpos_fk;
 *   UHC_MOTION_QPOS  qpos (pose_dim = 76): qpos_fk only (torch_smpl_humanoid.py:155-261).
 * The FK uses shape variant fk_model_host[c] of the engine's model for clip c (NULL = variant 0).  The records are computed in fp64 and
 * stored in the engine's precision.  The rows reach the device through a pinned staging buffer in chunks of whole clips of up to
 * chunk_frames frames (0 = 32768; a longer clip is a chunk of its own), so the device scratch is bounded by the chunk.  As after
 * uhc_load_clips: every env record is invalidated, the sampling weights return to the sample_keys rule and the clip models to
 * variant 0.  Clips shorter than 2 frames and arguments out of range are rejected (-2) with the previous table left loaded. */
#define UHC_MOTION_SMPL 0   /* rows: pose_aa (72 | 156) then trans (3) */
#define UHC_MOTION_QPOS 1   /* rows: qpos (76) */
int uhc_load_motions(UhcEngine *e, int nclips, const int *clip_len_host, int kind, int pose_dim, const double *rows_host,
                     const double *shape_host, const int *fk_model_host, int chunk_frames);
/* rows first .. first + n - 1 of clip `clip` of the loaded table, as doubles: out_host = [n][UHC_EX_SIZE] */
int uhc_get_clip_frames(UhcEngine *e, int clip, int first, int n, double *out_host);
/* device time of the last uhc_load_motions, from CUDA events (ms): out2[0] = its kernels, out2[1] = its host-to-device row copies */
int uhc_load_motions_time(const UhcEngine *e, float *out2);

/* body-shape variant of every clip (index into the model's shape variants); the reference rebuilds the robot per clip from
 * its beta/gender (humanoid_im.py:154-180).  Call after uhc_load_clips; default = variant 0 for every clip. */
int uhc_set_clip_models(UhcEngine *e, int nclips, const int *clip_model);

/* standing-neutral pose of the reactive starts (sample_data/standing_neutral.pkl: qpos[76], qvel[75]; humanoid_im.py:66,86,1269-1271). */
int uhc_set_neutral_pose(UhcEngine *e, const double *qpos76, const double *qvel75);

/* Clip sampling weights of the in-kernel re-seeding.  Default (weights_host == NULL, and after every uhc_load_clips) = the
 * sample_keys rule used when no success history exists (len // t_max + 1 copies per clip, dataset_amass_single.py:138-142,180-182).
 * The training loop of the reference passes its per-clip success history instead (agent_copycat.py:511-517): with probability
 * sampling_freq the clip is drawn from exp(-ewma(success)/temp), else uniformly (dataset_amass_single.py:183-186, math_utils.py:25-29);
 * the caller folds both into one weight per clip: w = sampling_freq * p_fail + (1 - sampling_freq) / C. */
int uhc_set_clip_weights(UhcEngine *e, int nclips, const float *weights_host);

/* env.reset() for n envs (mujoco_env.py:95-104 + humanoid_im.py:1245-1299).  clip/start/len select the expert slice
 * (dataset_amass_single.py:200-253); q/v override (may be NULL) = [n][76]/[n][75] floats on the device.
 * obs_dev = [num_envs][657] (rows of the listed envs are written). */
int uhc_env_reset(UhcEngine *e, int n, const int *env_ids_host, const int *clip_host, const int *start_host, const int *len_host,
                  const float *qpos_dev, const float *qvel_dev, float *obs_dev, void *stream);

/* env.step(a) for ALL envs (humanoid_im.py:1192-1243) fused with custom_reward (reward_function.py:12-88):
 * actions_dev [E][105] -> obs_dev [E][657], reward_dev [E], cinfo_dev [E][5], fail/end [E] (int32), percent [E];
 * torque_dev (optional) [E][15][69] = the per-substep torques (env.curr_torque). */
int uhc_env_step(UhcEngine *e, const float *actions_dev, float *obs_dev, float *reward_dev, float *cinfo_dev, int *fail_dev,
                 int *end_dev, float *percent_dev, float *torque_dev, void *stream);

/* Host-buffer convenience used by the single-env facade and the end-to-end benchmark: copies in/out inside the call. */
int uhc_env_step_host(UhcEngine *e, const float *actions_host, float *obs_host, float *reward_host, float *cinfo_host,
                      int *fail_host, int *end_host, float *percent_host);

/* parity hooks / fail_safe (humanoid_im.py:902-905): read or overwrite the simulator state of one env (host doubles). */
int uhc_env_get_state(UhcEngine *e, int env, double *qpos76, double *qvel75, double *xpos72, double *bquat96, int *istate8);
int uhc_env_set_state(UhcEngine *e, int env, const double *qpos76, const double *qvel75);
/* the same for n envs with one launch and one copy: out_host = [n][319] doubles (qpos76 qvel75 xpos72 bquat96), istate_host = [n][8]
 * (cur_t, clip, start, len, episode, flags (bit 0: contact overflow), newton iterations, max contacts); set: qpos [n][76], qvel [n][75]. */
int uhc_env_get_state_batch(UhcEngine *e, int n, const int *env_ids_host, double *out_host, int *istate_host);
int uhc_env_set_state_batch(UhcEngine *e, int n, const int *env_ids_host, const double *qpos_host, const double *qvel_host);
/* device counters: out4[0] = env-steps FAILED because a body's floor contacts did not fit the per-env contact capacity (40; MuJoCo's
 * generated models allocate nconmax 500, skeleton_mesh.py:46 -- such a step sets fail instead of continuing on a truncated contact
 * set), out4[1] = env-steps skipped because the env record was stale (clip table reloaded) or never reset (outputs: fail = end = 1). */
int uhc_engine_counters(UhcEngine *e, int *out4);
/* device array [E][2] written by every uhc_env_step: clip index of the episode that ended in that step (-1 = none) and its completed
 * fraction `percent` as float bits -- what the reference appends to its per-clip success history (agent_copycat.py:561). */
const int *uhc_episode_log_dev(const UhcEngine *e);
int uhc_num_envs(const UhcEngine *e);
int uhc_engine_obs_dim(const UhcEngine *e);      /* env.obs_dim (humanoid_im.py:256-258) */
int uhc_engine_act_dim(const UhcEngine *e);      /* env.action_dim (humanoid_im.py:250): 69 + (6 | 216) + (30 if meta_pd) */
int uhc_kernel_launches(const UhcEngine *e);   /* kernels launched by this engine so far (bench `gpu_launches`) */

#ifdef __cplusplus
}
#endif
#endif
