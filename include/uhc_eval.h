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
 * (uhc_eval_last_error()).  The call returns after its last copy has landed.
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

const char *uhc_eval_last_error(void);

/* Envs 0..n-1 are reset onto clips clip_host[0..n-1] from frame 0 (envs n..E-1 are parked on clip_host[0]), then stepped with the
 * deterministic policy (the mean action; zfilter_stats are read, not updated) for up to max(len) - 1 control steps under the engine's
 * current cfg (auto_reset off: the test-mode cfg).  After every step each env still alive records one frame row; an env stops after
 * `end`, and after `fail` unless fail_safe != 0, which re-seats it on the expert qpos / qvel of frame min(cur_t, len - 1) exactly as
 * uhc_env_set_state_batch does.  The steps run as a CUDA graph of `window` steps captured once per argument set and replayed.
 * frames_host = [n][max(len) - 1][UHC_EVAL_NCOL]: rows past an env's `frames` are unspecified.  clips_host = [n].
 * states_host_or_null = [n][max(len) - 1][UHC_EVAL_STATE] (parity tests; NULL costs nothing).  Bad arguments (-2): n < 1 or n > E,
 * a clip index out of range, no clip table loaded, window < 1, a policy whose widths are not the engine's obs / action dims. */
int uhc_eval_run(UhcEngine *e, int n, const int *clip_host, const UhcMlp *mlp, const float *log_std, const double *zfilter_stats, float zclip,
                 int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream);
int uhc_eval_run_mcp(UhcEngine *e, int n, const int *clip_host, const UhcMcp *mcp, const float *log_std, const double *zfilter_stats, float zclip,
                     int fail_safe, int window, double *frames_host, UhcEvalClip *clips_host, double *states_host_or_null, void *stream);
void uhc_eval_release(UhcEngine *e);   /* frees the graphs / scratch of this engine; call before uhc_engine_destroy */

#ifdef __cplusplus
}
#endif
#endif
