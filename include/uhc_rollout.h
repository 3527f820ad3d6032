/* uhc_rollout.h -- C ABI of the sampling loop (part of libuhc_b200.so): policy forward and the fused T-step rollout.
 *
 * Reference interface replaced (SURVEY.md section 8b lists these as the surface a C-ABI replacement must export):
 *   uhc_policy_forward   Agent.trans_policy + running_state + PolicyGaussian.select_action
 *                        (uhc/agents/agent_copycat.py:521-531, khrylib/rl/core/policy.py:12-15, policy_gaussian.py:26-31, utils/zfilter.py:59-73)
 *   uhc_rollout          AgentCopycat.sample_worker's loop body over all environments (uhc/agents/agent_copycat.py:496-571): per control step
 *                        normalise -> policy -> sample -> env.step -> custom_reward -> push(state, action, mask, reward, exp); finished
 *                        episodes are re-seeded inside the step kernel (UhcEnvCfg.auto_reset, :503-517 + dataset_amass_single.py:172-253).
 * All pointers are CUDA device pointers owned by the caller (PyTorch tensors: weights, ZFilter statistics, rollout buffer) unless
 * suffixed _host.  Calls are stream-ordered on `stream`; return 0 on success, <0 on error (uhc_last_error()).
 */
#ifndef UHC_ROLLOUT_H
#define UHC_ROLLOUT_H
#include "uhc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* MLP trunk + head in the tensor-core layout (khrylib/models/mlp.py:5-27 + PolicyGaussian.action_mean): layer i maps dims[i] -> dims[i+1];
 * W_bf16[i] = [dims[i+1]][kp[i]] bf16, kp[i] = dims[i] rounded up to 64 and zero padded; bias[i] fp32; act = UHC_ACT_* of the trunk. */
typedef struct {
    int nlayers, act;
    int dims[10];
    int kp[8];
    const void *W_bf16[8];
    const float *bias[8];
} UhcMlp;

/* PolicyMCP (uhc/models/policy_mcp.py:9-37, actor_type "mcp" of config/release/uhc_implicit.yml): nprim primitive MLPs (same widths as a
 * PolicyGaussian trunk + action_mean head) and a composer MLP obs -> composer_dim -> nprim whose EVERY layer is followed by the activation
 * (mlp.py:24-27) before the softmax; action_mean = sum_k softmax(composer(x))_k * prim_k(x). */
#define UHC_MCP_MAX_PRIM 8
typedef struct {
    int nprim, reserved;
    UhcMlp prim[UHC_MCP_MAX_PRIM];
    UhcMlp composer;
} UhcMcp;

/* Time-major rollout buffer [T_cap][E][...] (the device-resident TrajBatch, khrylib/rl/core/trajbatch.py:4-15) and the current
 * observation of every env (written by uhc_env_reset / the step kernel). logp / fails may be NULL. */
typedef struct {
    float *states, *actions, *rewards, *masks, *exps, *logp;
    int *fails;
    float *obs_cur;       /* [E][uhc_engine_obs_dim] raw observation before the step; overwritten with the next one */
    int *ep_clip;         /* optional [T_cap][E]: clip index of the episode that ended at this step (-1: none) ... */
    float *ep_pct;        /* ... and its completed fraction: the per-clip success history of agent_copycat.py:561 */
    int T_cap, reserved;
    int *ep_start;        /* optional [T_cap][E] (with ep_clip): the start frame of that episode (fr_start of agent_copycat.py:561), recorded while
                           * the device curriculum is enabled (its step-kernel variant logs it), -1 before it ever was */
} UhcRolloutBuf;

/* The failure-weighted curriculum on the device (the training loop's freq_dict, agent_copycat.py:561,590-603 + dataset_amass_single.py:172-232).
 * uhc_curriculum_enable allocates a ring of the last max_freq (percent, start) outcomes per clip, empty, and from then on owns the
 * sampler's clip CDF: uhc_set_clip_weights returns -2 while it is enabled.  Called again with the same max_freq it keeps the history and
 * only changes the parameters; max_freq = 0 disables it (the CDF returns to the sample_keys rule).  temp / freq = sampling_temp /
 * sampling_freq of the clip mixture; prec_freq = probability of a precision-mode start (0 = off; the reference's precision_mode passes
 * sampling_freq, or 0.75 with fit_single_key); fit_clip = -1, or the clip every re-seed uses.  A clip-table load with another clip count
 * disables the curriculum.  Bad arguments return -2 and leave the engine as it was. */
int uhc_curriculum_enable(UhcEngine *e, int max_freq, double temp, double freq, double prec_freq, int fit_clip);
/* After a rollout, on `stream`, without a host synchronise: appends the ended episodes of rows 0 .. T-1 of buf (ep_clip, ep_pct, ep_start
 * all required), step-major then env-minor, keeps each clip's last max_freq, and rewrites the clip CDF in place from the new weights
 * (the sample_keys rule while every history is empty). */
int uhc_curriculum_update(UhcEngine *e, const UhcRolloutBuf *buf, int T, void *stream);
/* One history across the ranks of a data-parallel run, carried by the gradient all-reduce (uhc_ppo_update_ex's extra payload):
 * uhc_curriculum_stage zeroes `slots` ([world][T][E][3] fp32, world * T * E * 3 floats) and writes rows 0 .. T-1 of buf (ep_clip, ep_pct, ep_start
 * all required) into slot `rank` as (clip, percent, start), (-1, 0, 0) where no episode ended.  Summed over the ranks, the slots are every rank's
 * log exactly (every element is one rank's value plus zeros).  uhc_curriculum_update_gathered unpacks such a sum into one log of world * T * E
 * entries, rank-major, then step-major, then env-minor, and appends it as uhc_curriculum_update does: after it every rank holds the rings and the
 * CDF one curriculum fed with every rank's log would hold.  Stream-ordered, no host synchronise.  Both return -2 for bad arguments and when a
 * clip index or a start frame could exceed 2^24 (more than 2^24 clips, or a clip longer than 2^24 frames), where fp32 stops being exact. */
int uhc_curriculum_stage(UhcEngine *e, const UhcRolloutBuf *buf, int T, int rank, int world, float *slots, void *stream);
int uhc_curriculum_update_gathered(UhcEngine *e, const float *summed_slots, int T, int world, void *stream);
/* host-side history: append n outcomes in order (eval results); read / replace every clip's history, oldest first:
 * len_host [C], pct_host / start_host [C][max_freq] (entries past len[c] are ignored / zero).  Each updates the CDF. */
int uhc_curriculum_push(UhcEngine *e, int n, const int *clip_host, const float *pct_host, const int *start_host);
int uhc_curriculum_get(UhcEngine *e, int *len_host, float *pct_host, int *start_host);
int uhc_curriculum_set(UhcEngine *e, const int *len_host, const float *pct_host, const int *start_host);
/* re-seeds every env through the in-kernel sampler (a fit_clip change takes effect at once); obs_dev [E][obs_dim] gets the reset rows */
int uhc_curriculum_reseed(UhcEngine *e, float *obs_dev, void *stream);

const char *uhc_rollout_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* RNG stream position of the action noise: element (step, env, dim) of the stream `seed`; advanced by one per rollout step. */
int uhc_rollout_set_step(UhcEngine *e, unsigned long long step);
int uhc_rollout_get_step(UhcEngine *e, unsigned long long *step);

/* obs [E][657] -> ZFilter (update_filter != 0 merges the batch into zfilter_stats first) -> MLP on tensor cores -> Gaussian head:
 * action = mean + exp(log_std) eps (the mean where mean_action[e] != 0), logp = summed Normal log-prob.  state_out = the normalised
 * observation (what the reference pushes into its memory), may be NULL.  Does not advance the step counter. */
int uhc_policy_forward(UhcEngine *e, const float *obs_dev, const UhcMlp *mlp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                       unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                       void *stream);

/* the same with a PolicyMCP mixture in place of the single MLP */
int uhc_policy_forward_mcp(UhcEngine *e, const float *obs_dev, const UhcMcp *mcp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                           unsigned long long seed, const unsigned char *mean_action_or_null, float *state_out_or_null, float *action_out, float *logp_out_or_null,
                           void *stream);

/* T lock-step control steps of every env into rows row0 .. row0+T-1 of the buffer.  noise_rate: P(sampled action) per env and step
 * (agent_copycat.py:530; exp = 1 for sampled rows).  use_graph != 0: the kernel sequence is captured once per argument set into a
 * CUDA graph and replayed (no host work between kernels); 0: plain stream launches of the same kernels (bit-identical results). */
int uhc_rollout(UhcEngine *e, int T, int row0, const UhcMlp *mlp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream);
int uhc_rollout_mcp(UhcEngine *e, int T, int row0, const UhcMcp *mcp, const float *log_std, double *zfilter_stats, float zclip, int update_filter,
                    unsigned long long seed, float noise_rate, const UhcRolloutBuf *buf, int use_graph, void *stream);
/* measurement hook: CUDA events around the env-step kernel of buffer rows 0 .. nrows-1, recorded on the launching stream (also inside
 * graph replays); uhc_rollout_env_step_ms returns the duration of the last step written to `row`.  nrows = 0 disables. */
int uhc_rollout_time_env_step(UhcEngine *e, int nrows);
int uhc_rollout_env_step_ms(UhcEngine *e, int row, float *ms);
int uhc_rollout_launches_per_step(UhcEngine *e);   /* kernels per control step of the last uhc_rollout (bench `gpu_launches`) */
void uhc_rollout_release(UhcEngine *e);            /* frees graphs / scratch of this engine; optional: uhc_engine_destroy frees it too */

#ifdef __cplusplus
}
#endif
#endif
