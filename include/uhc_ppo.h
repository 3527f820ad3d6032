/* uhc_ppo.h -- C ABI of the PPO update: the whole of `agent.update` behind one call.
 *
 * Replaces (reference file:line under /root/reference):
 *   AgentPG.update_params          uhc/khrylib/rl/agents/agent_pg.py:39-56     V(s), estimate_advantages, update_policy
 *   estimate_advantages            uhc/khrylib/rl/core/common.py:5-25          GAE + advantage normalisation
 *   AgentPPO.update_policy         uhc/khrylib/rl/agents/agent_ppo.py:16-51    per epoch: value step (agent_pg.py:18-25), clipped-surrogate policy step
 *   AgentPPO.ppo_loss / clip_grad  uhc/khrylib/rl/agents/agent_ppo.py:53-65
 *   torch.optim.Adam steps         uhc/agents/agent_copycat.py:160-177
 * Multi-GPU (envs sharded by rank, SURVEY.md section 8e): the ONLY collective is the all-reduce(sum) of each net's flat gradient tensor per
 * optimisation step, issued on the caller's ncclComm_t from a side stream so it overlaps the other net's forward / backward; the
 * global-batch statistics (advantage moments and count, selected-row count, the ranks' ZFilter increments) ride in the tail of the first one.
 *
 * Every GEMM runs on the wgmma kernel (bf16 operands, fp32 accumulate; mlp_wgmma.cu); parameters, gradients and Adam moments are fp32.
 * All pointers are device pointers unless marked host.  Functions return 0 on success; uhc_last_error() describes the last failure.
 */
#ifndef UHC_PPO_H
#define UHC_PPO_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

/* one MLP (khrylib/models/mlp.py:5-27 + its linear head) with flat fp32 storage */
typedef struct UhcNetDesc {
    int nlayers, act;          /* Linear layers incl. the head (<= 8); hidden activation UHC_ACT_* (uhc_nn.h) */
    int dims[10];              /* dims[0] = input width ... dims[nlayers] = output width */
    float *flat;               /* parameters: W[i] ([dims[i+1]][dims[i]], row-major) at w_off[i], b[i] at b_off[i] */
    float *gfull;              /* gradients in the same layout, followed by `gtail` floats (statistics riding the all-reduce) */
    long nflat, gtail;
    long w_off[8], b_off[8];
    float *adam_m, *adam_v;    /* Adam moments, nflat floats each */
    float lr;
    void *W_bf16[8];           /* bf16 copies of W[i] with K padded to kp[i] = dims[i] rounded up to 64: refreshed IN PLACE after every step */
    int kp[8];
    int head_act;              /* activation after the OUTPUT layer: UHC_ACT_NONE for policy / value heads, the trunk's activation for a PolicyMCP composer */
} UhcNetDesc;

typedef struct UhcPpoCfg {
    float gamma, tau, clip_eps;
    float grad_clip;               /* clip_grad_norm_ threshold of the policy step */
    int clip_first_step_only;      /* the reference passes a consumed generator to clip_grad_norm_ after the first policy step of a run
                                      (agent_copycat.py:93): != 0 clips only when *policy_steps_done == 0; 0 clips every policy step */
    int epochs;                    /* num_optim_epoch */
} UhcPpoCfg;

typedef struct UhcPpoTrainer UhcPpoTrainer;

const char *uhc_ppo_last_error(void);   /* an alias of uhc_last_error (uhc_b200.h): the library keeps one error text */

/* workspace for updates of up to max_rows transitions from up to max_envs environments (both nets, shared backward scratch) */
int uhc_ppo_trainer_create(const UhcNetDesc *policy, const UhcNetDesc *value, long max_rows, int max_envs, int device, UhcPpoTrainer **out);
/* PolicyMCP (uhc/models/policy_mcp.py:9-37): policy_nets = nprim primitive nets followed by the composer (head_act = its activation).  Every
 * entry shares ONE flat parameter / gradient / Adam tensor (flat, gfull, adam_m, adam_v, nflat identical; w_off / b_off are offsets into it), so the
 * mixture is still one all-reduce and one Adam launch per step. */
int uhc_ppo_trainer_create_mcp(const UhcNetDesc *policy_nets, int nprim, const UhcNetDesc *value, long max_rows, int max_envs, int device, UhcPpoTrainer **out);
void uhc_ppo_trainer_destroy(UhcPpoTrainer *t);

/* The collective the trainer's updates with world > 1 call: ncclAllReduce's signature, the stream passed as a void *.  The trainer calls it in
 * place (sendbuff == recvbuff) with datatype 7 (ncclFloat32) and op 0 (ncclSum); a non-zero return fails the update. */
typedef int (*UhcAllReduceFn)(const void *sendbuff, void *recvbuff, size_t count, int datatype, int op, void *comm, void *stream);
/* installs fn as this trainer's all-reduce (another process-group implementation, or an in-process one for tests); NULL restores the default,
 * ncclAllReduce from libnccl.so.2 */
int uhc_ppo_trainer_set_all_reduce(UhcPpoTrainer *t, UhcAllReduceFn fn);

/* One PPO iteration's update on a time-major [T][E] rollout (M = T*E rows, row = t*E + e):
 *   states [M][dims[0]] normalised observations, last_states [E][dims[0]] the normalised observation after the last step (bootstrap V(s_T)),
 *   actions [M][A], rewards / masks / exps [M], log_std [A].
 *   adam_step_policy / adam_step_value (host, in/out): optimiser step counters; policy_steps_done (host, in/out): policy steps of this run so far.
 *   zfilter_stats / zfilter_sync (world > 1, may be NULL when world == 1): the running observation statistics [n, mean[D], S[D]] of this rank and
 *   the additive form [n, sum, sumsq] of what every rank agreed on last; on return every rank holds the merged statistics.
 *   nccl_comm: ncclComm_t of the training job (NULL = single GPU); world = its size.  Every rank must pass the same T and E: the value
 *   gradient is scaled by 1 / (T E world), and ranks whose gradient tensors differ in length cannot all-reduce them.
 *   losses_out (device, 2 floats): clipped-surrogate loss and value loss of the last epoch.  world == 1: the batch's means; world > 1: this
 *   rank's share of the global means (their sum over the ranks is the global loss; nothing sums it). */
int uhc_ppo_update(UhcPpoTrainer *t, const float *states, const float *last_states, const float *actions, const float *rewards, const float *masks,
                   const float *exps, const float *log_std, int T, int E, const UhcPpoCfg *cfg, int *adam_step_policy, int *adam_step_value,
                   int *policy_steps_done, double *zfilter_stats, double *zfilter_sync, void *nccl_comm, int world, float *losses_out, void *stream);
/* uhc_ppo_update with an extra payload on the same collective: the n_extra device floats at extra_in ride behind the statistics in the value
 * gradient's tail, and right after the first value all-reduce their sum over the ranks is copied to extra_out (world == 1: extra_in itself).
 * With world > 1 the value net's gtail must hold 5 (5 + 2 dims[0]) + n_extra floats, or the call returns -2.  The payload changes no gradient
 * element: it only lengthens the tail.  n_extra == 0 is uhc_ppo_update (the global curriculum's payload: uhc_curriculum_stage, uhc_rollout.h). */
int uhc_ppo_update_ex(UhcPpoTrainer *t, const float *states, const float *last_states, const float *actions, const float *rewards, const float *masks,
                      const float *exps, const float *log_std, int T, int E, const UhcPpoCfg *cfg, int *adam_step_policy, int *adam_step_value,
                      int *policy_steps_done, double *zfilter_stats, double *zfilter_sync, void *nccl_comm, int world, float *losses_out,
                      const float *extra_in, float *extra_out, long n_extra, void *stream);

/* AgentPPO.update_policy (agent_ppo.py:16-51) alone: the epochs on caller-provided returns and (already normalised) advantages, M rows.
 * Single GPU only: world > 1 returns -2 (the selected-row count it would divide the policy gradient by is this rank's, not the global one). */
int uhc_ppo_update_policy(UhcPpoTrainer *t, const float *states, const float *actions, const float *returns, const float *advantages, const float *exps,
                          const float *log_std, long M, const UhcPpoCfg *cfg, int *adam_step_policy, int *adam_step_value, int *policy_steps_done,
                          void *nccl_comm, int world, float *losses_out, void *stream);

/* advantages / returns of the last update (device, M floats each; valid until the next call) -- parity hooks */
const float *uhc_ppo_advantages(const UhcPpoTrainer *t);
const float *uhc_ppo_returns(const UhcPpoTrainer *t);
long uhc_ppo_kernel_launches(const UhcPpoTrainer *t);   /* kernels enqueued by uhc_ppo_update so far (bench `gpu_launches`) */
/* collectives of the calls so far: total milliseconds (CUDA events on the side stream; synchronises it), bytes, calls; resets the counters */
int uhc_ppo_comm_stats(UhcPpoTrainer *t, double *ms, long *bytes, int *calls);

#ifdef __cplusplus
}
#endif
#endif
