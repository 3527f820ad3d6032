/* uhc_eval.h -- C ABI of the device evaluation (part of libuhc_b200.so): deterministic roll-outs of whole clips with fail-safe and
 * per-frame imitation metrics, one call per chunk of at most E clips.
 *
 * Reference interface replaced: the chunk loop of AgentCopycat.eval_policy (uhc/agents/agent_copycat.py, the host loop this library
 * keeps as the default) -- per control step running_state -> policy mean -> env.step, a state read of every live env, fail_safe
 * re-seats (humanoid_im.py:902-905) and, after the loop, smpl_eval.compute_metrics per clip (uhc_b200/metrics.py).  Here the steps
 * run as CUDA-graph replays with the metrics computed on the device (uhc_b200/csrc/eval_core.h); the host sees one frame-row copy and
 * one "any env alive" count per `window` steps.
 * Pointers suffixed _host are host memory (frames_host / states_host should be pinned: their copies are asynchronous); the others are
 * CUDA device pointers (PyTorch tensors).  Returns 0 on success, -2 on a bad argument (the engine stays usable), -1 on a CUDA error
 * (uhc_last_error()).  The call returns after its last copy has landed.
 */
#ifndef UHC_EVAL_H
#define UHC_EVAL_H
#include "uhc_b200.h"
#include "uhc_rollout.h"
#ifdef __cplusplus
extern "C" {
#endif

/* per env of one call */
typedef struct {
    int frames;          /* frames recorded = control steps while the env was alive */
    int last_t;          /* cur_t after the last recorded step (info["percent"] numerator) */
    int fail_any;        /* the env failed at least once (fail_safe re-seats it; otherwise it stopped there) */
    int reserved;
    double reward_sum;   /* fp32 rewards of the recorded steps summed in fp64 in step order */
} UhcEvalClip;

/* per-frame columns of frames_host (uhc_b200/csrc/eval_core.h): mpjpe_g, mpjpe, pa_mpjpe (mm), vel (mm, valid from frame 1),
 * accel (mm, valid from frame 2), |I - X_pred X_gt^-1|_F (root_dist_mm before its / T * 1000) */
#define UHC_EVAL_NCOL 6
/* states_host columns: the recorded qpos (76) and world body positions xpos (72) of every frame, as doubles */
#define UHC_EVAL_STATE 148
/* smpl_host columns: the recorded qpos as SMPL (include/uhc_export.h uhc_qpos_to_smpl), pose 72 (axis-angle, SMPL_BONE_ORDER_NAMES order)
 * then trans 3, as doubles */
#define UHC_EVAL_SMPL 75

/* the outputs of one evaluation call (the _ex entry points) */
typedef struct {
    double *frames_host;           /* [n][max(len) - 1][UHC_EVAL_NCOL] */
    UhcEvalClip *clips_host;       /* [n] */
    double *states_host_or_null;   /* [n][max(len) - 1][UHC_EVAL_STATE] */
    double *smpl_host_or_null;     /* [n][max(len) - 1][UHC_EVAL_SMPL] */
    double *floor_host_or_null;    /* [n][max(len) - 1][UHC_FLOOR_NCOL] (include/uhc_floor.h) */
} UhcEvalOut;

const char *uhc_eval_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* Envs 0..n-1 are reset onto clips clip_host[0..n-1] from frame 0 (envs n..E-1 are parked on clip_host[0]), then stepped with the
 * deterministic policy (the mean action; zfilter_stats are read, not updated) for up to max(len) - 1 control steps under the engine's
 * current cfg (auto_reset off: the test-mode cfg).  After every step each env still alive records one frame row; an env stops after
 * `end`, and after `fail` unless fail_safe != 0, which re-seats it on the expert qpos / qvel of frame min(cur_t, len - 1) exactly as
 * uhc_env_set_state_batch does.  The steps run as a CUDA graph of `window` steps captured once per argument set and replayed.
 * frames_host = [n][max(len) - 1][UHC_EVAL_NCOL]: rows past an env's `frames` are unspecified.  clips_host = [n].
 * states_host_or_null = [n][max(len) - 1][UHC_EVAL_STATE] (parity tests; NULL costs nothing).  Bad arguments (-2): n < 1 or n > E,
 * a clip index out of range, no clip table loaded, window < 1 or n * window > INT_MAX, a policy whose widths are not the engine's obs / action dims. */
int uhc_eval_run(UhcEngine *e, int n, const int *clip_host, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats, float zclip,
                 int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream);
int uhc_eval_run_mcp(UhcEngine *e, int n, const int *clip_host, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats, float zclip,
                     int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream);
/* Several policies of one architecture in one call (checkpoint sweeps): group g owns envs [off_g, off_g + n_g), off_g = sum_{h<g} n_h,
 * sum n_g <= E, and runs policy mlps[g] (mcps[g]) with its own ZFilter statistics zfilter_stats_host[g] (a host array of G device pointers)
 * on clips clip_host[off_g .. off_g + n_g - 1].  Everything else is uhc_eval_run over the sum n of the group sizes: frames_host = [n][max(len) - 1]
 * [UHC_EVAL_NCOL] with max(len) over every listed clip, clips_host = [n], states_host_or_null = [n][max(len) - 1][UHC_EVAL_STATE]; envs past
 * the last group are parked on clip_host[0] and step with zero actions.  Each group's rows are bit-identical to a uhc_eval_run of its own
 * policy on its own clips (with any finite log_std: the mean action needs none).  The policy GEMMs of all groups run as one grouped
 * tensor-core launch per layer.  Bad arguments (-2, the engine stays usable): G < 1 or G > UHC_EVAL_MAX_GROUPS, an n_g < 1, sum n > E, a clip
 * out of range, no clip table, window < 1, a null policy or statistics pointer, policies whose layer widths, K padding, activation or
 * primitive count differ between groups, widths that are not the engine's obs / action dims. */
#define UHC_EVAL_MAX_GROUPS 64
int uhc_eval_run_groups(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMlp *mlps, const double *const *zfilter_stats_host,
                        float zclip, int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream);
int uhc_eval_run_groups_mcp(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMcp *mcps, const double *const *zfilter_stats_host,
                            float zclip, int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream);
/* The four calls above with their outputs in one UhcEvalOut, which adds the SMPL export: with out->smpl_host_or_null set, each recorded frame's
 * qpos -- the stepped state before any fail_safe re-seat, the state record's qpos -- is converted on the device by uhc_qpos_to_smpl's code with
 * the shape variant of the env's clip, and row [i][f] of smpl_host equals uhc_qpos_to_smpl of row [i][f] of states_host bit for bit.  Rows past
 * an env's `frames` are unspecified.  With smpl_host_or_null = NULL each is the call above (the same graph and outputs); the graphs with and
 * without the export are cached side by side.
 * With out->floor_host_or_null set (after uhc_floor_init, include/uhc_floor.h; -2 without it) each recorded frame's hulls are measured against
 * the floor on the device from the same recorded state: row [i][f] of floor_host equals uhc_floor_qpos of rows f - 1, f of states_host[i]
 * (row 0 without a previous frame) bit for bit.  NULL costs nothing: the graph, its outputs and its cache entry are those without the field. */
int uhc_eval_run_ex(UhcEngine *e, int n, const int *clip_host, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats, float zclip,
                    int fail_safe, int window, const UhcEvalOut *out, void *stream);
int uhc_eval_run_mcp_ex(UhcEngine *e, int n, const int *clip_host, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats, float zclip,
                        int fail_safe, int window, const UhcEvalOut *out, void *stream);
int uhc_eval_run_groups_ex(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMlp *mlps, const double *const *zfilter_stats_host,
                           float zclip, int fail_safe, int window, const UhcEvalOut *out, void *stream);
int uhc_eval_run_groups_mcp_ex(UhcEngine *e, int G, const int *group_n_host, const int *clip_host, const UhcMcp *mcps, const double *const *zfilter_stats_host,
                               float zclip, int fail_safe, int window, const UhcEvalOut *out, void *stream);
int uhc_eval_graph_count(const UhcEngine *e);   /* graphs this engine's evaluation holds now, grouped ones included (read-only; tests) */
void uhc_eval_release(UhcEngine *e);   /* frees the graphs / scratch of this engine (the grouped path's too); optional: uhc_engine_destroy frees it too */

#ifdef __cplusplus
}
#endif
#endif
