/* uhc_track.h -- C ABI of the batched physics tracker (part of libuhc_b200.so): the trained controller follows target poses that are
 * streamed one frame per control step, for all envs at once.
 *
 * Reference interface replaced: HumanoidKinEnv.step (uhc/envs/humanoid_kin_v1.py:297-370) -- per step a kinematic model produces the next
 * target qpos, qpos_fk turns it into the target frame, the cc policy's mean action on the cc obs against that frame drives do_simulation.
 * Here the caller streams the raw target frames (device memory), the engine turns each into an expert-table record on the device
 * (the records of uhc_load_motions, bit for bit) and one CUDA-graph replay per call runs observation, policy, physics and fail_safe.
 *
 * Tracking mode owns the engine's clip table: env e follows clip e, a window of H rows.  A later uhc_load_clips / uhc_load_motions ends
 * it (uhc_track_step then returns -2).  Pointers suffixed _dev are CUDA device pointers, _host host pointers.  Returns 0 on success,
 * -2 on a bad argument (the engine is left as it was), -1 on a CUDA error (uhc_last_error()).
 */
#ifndef UHC_TRACK_H
#define UHC_TRACK_H
#include "uhc_b200.h"
#include "uhc_rollout.h"
#include "uhc_subject.h"
#ifdef __cplusplus
extern "C" {
#endif

/* per env columns of uhc_track_state */
#define UHC_TRACK_STATE_COLS 4   /* control steps taken since the env's reset, cur_t in the window, rows held, pushes dropped (window full) */
/* columns of state_out_dev: qpos 76, qvel 75, world body positions xpos 72, in the engine's precision */
#define UHC_TRACK_OUT 223

const char *uhc_track_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* Installs a table of E clips x `window` rows (env e owns clip e) through the table set-up of uhc_load_clips: every env record is
 * invalidated, clip models = fk_model_host (NULL: variant 0; also the FK's shape variant), shape vectors = shape_host [E][17] (NULL: zero).
 * kind / pose_dim: the raw-row formats of uhc_load_motions (UHC_MOTION_QPOS 76, UHC_MOTION_SMPL 72 | 156; row width pose_dim + 3).
 * -2 for what a stream cannot serve: obs_v 3 (future frames), term_body root / Head (the whole episode window), auto_reset, reactive_v 1,
 * window < 3, and a cfg whose `end` could fire inside the window (needs trail_steps >= 1 and env_episode_len >= window). */
int uhc_track_begin(UhcEngine *e, int window, int kind, int pose_dim, const int *fk_model_host, const double *shape_host);
/* Frames 0 and 1 of each listed env's stream (frames_dev = [n][2][row width] fp64) become rows 0 and 1, then the env is reset onto row 0
 * exactly as uhc_env_reset does (qpos_dev / qvel_dev: optional fp32 overrides [n][76] / [n][75]).  Its step count returns to 0. */
int uhc_track_reset(UhcEngine *e, int n, const int *env_ids_host, const double *frames_dev, const float *qpos_dev, const float *qvel_dev, void *stream);
/* One control step of every env, in order: push frame t + 1 (next_frames_dev [E][row width] fp64, NULL = no push; mask_dev [E] int32,
 * NULL = all, 0 = this env gets no frame), the observation of each env's state against row cur_t + 1, ZFilter (no update) + policy mean,
 * k_env_step, fail_safe re-seat on row cur_t of the envs that failed.  state_out_dev [E][UHC_TRACK_OUT] = the state the step produced
 * (before a re-seat), reward_dev [E] fp32, fail_dev [E] int32.  An env whose row cur_t + 1 was never pushed is not stepped: fail = 1,
 * reward 0, counted in uhc_engine_counters' skipped steps.  The first call after a reset passes next_frames_dev = NULL (the reset pushed
 * frame 1).  Replays one CUDA graph per argument set; no host synchronise. */
int uhc_track_step(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, const UhcMlp *mlp, const float *log_std,
                   const double *zfilter_stats, float zclip, int fail_safe, void *state_out_dev, float *reward_dev, int *fail_dev, void *stream);
int uhc_track_step_mcp(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, const UhcMcp *mcp, const float *log_std,
                       const double *zfilter_stats, float zclip, int fail_safe, void *state_out_dev, float *reward_dev, int *fail_dev, void *stream);
/* the push of uhc_track_step on its own (frames known ahead of the steps); a push into a full window whose rows are all still needed is
 * dropped and counted (uhc_track_state column 3) */
int uhc_track_push(UhcEngine *e, const double *next_frames_dev, const int *mask_dev, void *stream);
/* the observation uhc_track_step feeds the policy, without stepping: obs_dev [E][obs dim], zero rows for envs it would not step */
int uhc_track_obs(UhcEngine *e, float *obs_dev, void *stream);
/* out_host = [E][UHC_TRACK_STATE_COLS] (synchronises the device) */
int uhc_track_state(UhcEngine *e, int *out_host);
/* frees the stream buffers and graphs; the clip table stays loaded (its rows are whatever the windows held) */
void uhc_track_end(UhcEngine *e);
/* CUDA graphs the tracker of this engine holds now (read-only; tests) */
int uhc_track_graph_count(const UhcEngine *e);

/* Run-time subjects: each env simulates and follows its own body, built on the device from SMPL beta and gender (include/uhc_subject.h), as
 * the reference rebuilds its humanoid for every sequence (HumanoidEnv.load_expert -> reset_robot).
 *
 * uhc_track_subjects_enable uploads `basis` (for the engine's variant 0) and, on the first call, reserves one extra shape variant per env,
 * slot nshape + env, in every per-variant table of the engine: body_f and hull in the engine's precision, the FK's fp64 body table, and the
 * hull in fp64 for the floor measurements.  Each slot starts as a copy of variant 0.  Memory: per env 24 x 20 + nvert x 3 values of the
 * engine's precision, 24 x 6 + nvert x 3 doubles.  The tables move, so the graphs of the rollout, the evaluation and the tracker captured
 * before are dropped, never replayed.  Call it before uhc_track_begin: -2 while tracking is active, or for a basis uhc_subject_bodies
 * refuses (nothing changes then); a later call replaces the basis and keeps the slots. */
int uhc_track_subjects_enable(UhcEngine *e, const UhcSubjectBasis *basis);
/* While tracking on an enabled engine: for each listed env, its body from beta[:10] and the gender (shape_host [n][17] = beta 16, gender code
 * 0 neutral / 1 male / 2 female), by uhc_subject_bodies' code, written into its slot of every table (the engine-precision values rounded as
 * uhc_engine_create rounds them); its clip model and FK variant become the slot, its shape observation the row, and its record is
 * invalidated: it is not stepped until uhc_track_reset builds its rows with the new body's FK.  The other envs are untouched, and tracker
 * steps replay the same graphs (the tables keep their addresses).  The call synchronises `stream` once, after the build: -2 with every table
 * as before for an inverted body (det A <= 0), and, with nothing launched, for env ids out of range or listed twice, a non-finite value, a
 * gender without a basis, or an engine that is not tracking or not enabled. */
int uhc_track_set_subjects(UhcEngine *e, int n, const int *env_ids_host, const double *shape_host, void *stream);
/* env's slot as the engine holds it, each output optional (NULL: skipped): body_f [24][20] and hull [nvert][3] in the engine's precision widened
 * to fp64, the FK's body rows [24][6] (offset, ipos) and the fp64 hull of the floor measurements [nvert][3].  Synchronises the device. */
int uhc_track_subject_tables(UhcEngine *e, int env, double *body_f_host, double *hull_host, double *fk_body_host, double *hull64_host);

#ifdef __cplusplus
}
#endif
#endif
