/* uhc_nn.h -- C ABI of the policy/value network, Gaussian head, observation normaliser, GAE and PPO-update kernels
 * (part of libuhc_b200.so).  All pointers are CUDA device pointers owned by the caller (PyTorch tensors hold the weights --
 * the checkpoint format of the reference is a torch state_dict, uhc/agents/agent_copycat.py:190-201); `stream` is a cudaStream_t.
 * Return 0 on success, <0 on error (uhc_last_error()).  Each entry cites the reference Python it replaces.
 */
#ifndef UHC_NN_H
#define UHC_NN_H
#ifdef __cplusplus
extern "C" {
#endif

enum { UHC_ACT_NONE = 0, UHC_ACT_GELU = 1, UHC_ACT_TANH = 2, UHC_ACT_RELU = 3, UHC_ACT_SIGMOID = 4 };  /* mlp.py:9-16 */

/* aliases of uhc_last_error (uhc_b200.h): the library keeps one error text, the tensor-core entry points included */
const char *uhc_nn_last_error(void);
const char *uhc_tc_last_error(void);

/* nn.Linear + activation (khrylib/models/mlp.py:24-27):  y[M][N] = act(x[M][K] W[N][K]^T + b[N]); z (optional) = pre-activation. */
int uhc_linear_forward(const float *x, const float *W, const float *b, float *y, float *z_or_null, int M, int N, int K, int act, void *stream);
/* autograd of the same layer: dx[M][K] = dz W ; dW[N][K] = dz^T x ; db[N] = colsum(dz).  dx may be NULL (first layer). */
int uhc_linear_backward(const float *x, const float *W, const float *dz, float *dx_or_null, float *dW, float *db, int M, int N, int K, void *stream);
int uhc_act_backward(const float *dh, const float *z, float *dz, long n, int act, void *stream);

/* tensor-core forward of the same layer for the rollout path (wgmma, bf16 operands, fp32 accumulate): see mlp_wgmma.cu.
 * x_bf16 [M][Kp], W_bf16 [N][Kp] with Kp a multiple of 64 (zero padded); y_bf16 [M][Np] (next layer's input) and/or y_f32 [M][N].
 * A bf16 y needs a 16-byte aligned base and a pitch ldy_bf16 >= N that is a multiple of 8 (every tensor-core entry point returns -2 otherwise,
 * the grouped one included); its columns N .. min(ldy, N rounded up to 128) are written as zeros. */
int uhc_linear_forward_tc(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16_or_null, float *y_f32_or_null,
                          int M, int N, int Kp, int ldy_bf16, int act, void *stream);
/* the same for G <= UHC_TC_MAX_GROUPS weight sets in one launch: rows [row0_host[g], row0_host[g] + rows_host[g]) of x and y use W_bf16_host[g]
 * and b_host[g] (host arrays of device pointers; b_host may be NULL, as may an entry).  The ranges must be non-empty, ascending, disjoint
 * and inside [0, M); rows outside every range are not written.  Each row's output is bit-identical to uhc_linear_forward_tc with its
 * group's weights (the row tiles of a launch never straddle two groups: uhc_b200/csrc/group_core.h). */
#define UHC_TC_MAX_GROUPS 64
int uhc_linear_forward_tc_grouped(int G, const int *row0_host, const int *rows_host, const void *x_bf16, const void *const *W_bf16_host,
                                  const float *const *b_host_or_null, void *y_bf16_or_null, float *y_f32_or_null, int M, int N, int Kp, int ldy_bf16,
                                  int act, void *stream);
int uhc_f32_to_bf16_padded(const float *x, void *y_bf16, int M, int K, int Kp, void *stream);
/* training variants on the tensor cores (bf16 operands, fp32 accumulate; autograd of nn.Linear + activation):
 *   forward that also stores the pre-activation z (fp32) ; dX = dZ W and dW = dZ^T X are plain calls of uhc_linear_forward_tc on
 *   transposed bf16 copies ; uhc_dact_bf16 fuses dz = dh * act'(z) -> bf16 dz, bf16 dz^T and the bias gradient. */
int uhc_linear_forward_tc_train(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16_or_null, float *y_f32_or_null, float *z_f32,
                                int M, int N, int Kp, int ldy_bf16, int act, void *stream);
/* the same, also emitting the transposed bf16 activation yT [N][ld_yT] (ld_yT >= M, multiple of 8, zero padded): the dW GEMM's K-major operand, stored by the
 * epilogue through the TMA engine.  Needs the TMA-store path (uhc_tc_tma_store_enabled(); UHC_TC_TMA_STORE=0 in the environment turns it off). */
int uhc_linear_forward_tc_train_t(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16, void *yT_bf16, int ld_yT, float *z_f32_or_null,
                                  int M, int N, int Kp, int ldy_bf16, int act, void *stream);
/* plain fp32 product y[M][ld_y] = x W^T with an explicit row pitch ld_y >= N (floats, multiple of 4, 16-byte aligned output) through the TMA engine, split-K
 * where the output has few tiles; -2 when the arguments are not eligible (or the TMA-store path is off) */
int uhc_linear_forward_tc_f32_pitched(const void *x_bf16, const void *W_bf16, float *y_f32, int ld_y, int M, int N, int Kp, void *stream);
int uhc_tc_tma_store_enabled(void);
/* backward through one Linear and the PREVIOUS layer's activation in one kernel: dz_prev = (dz W) * act'(z_prev), emitted as bf16 [M][ld_dz] and transposed
 * [K][ld_dzT] (zero padded), db_prev[k] = sum_m dz_prev[m][k]; no fp32 dh is written.  dz [M][Np], WT [K][Np] bf16 K-major.  Returns -2 when the shapes
 * do not allow the TMA path (K % 4 != 0, unaligned buffers, UHC_TC_TMA_STORE=0): use uhc_linear_forward_tc + uhc_dact_bf16 then. */
int uhc_linear_dx_dact_tc(const void *dz_bf16, const void *WT_bf16, const float *z_prev, void *dzp_bf16, void *dzpT_bf16, float *db_prev_or_null,
                          int M, int K, int Np, int ld_dz, int ld_dzT, int act, void *stream);
int uhc_transpose_bf16(const void *in, void *out, int R, int C, int ld_in, int ld_out, void *stream);
int uhc_dact_bf16(const float *dh, const float *z_or_null, void *dz_bf16, void *dzT_bf16, float *db_or_null, int M, int N, int ld_dz, int ld_dzT, int act,
                  void *stream);

/* DiagGaussian (khrylib/rl/core/distributions.py:6-25, policy.py:12-23): sample a = mean + exp(log_std) eps (or the mean where
 * mean_action[i] != 0), log-prob summed over the action dims. */
int uhc_gaussian_sample(const float *mean, const float *log_std, const unsigned char *mean_action, float *action, float *logp, int M, int A,
                        unsigned long long seed, unsigned long long step, void *stream);
int uhc_gaussian_logprob(const float *mean, const float *log_std, const float *action, float *logp, int M, int A, void *stream);

/* PolicyMCP mixture head (uhc/models/policy_mcp.py:28-36): mean = sum_k softmax(c)_k xall_k ; xall = [P][M][A] primitive outputs, c = [M][P] composer
 * outputs (after the composer MLP's last activation); weight [M][P] = the softmax, kept for uhc_mcp_backward, which returns the gradients wrt
 * the primitive outputs (dxall [P][M][A]) and wrt c (dc [M][P]) given dmean. */
int uhc_mcp_combine(const float *xall, const float *c, float *weight_or_null, float *mean, int M, int A, int P, void *stream);
int uhc_mcp_backward(const float *xall, const float *weight, const float *dmean, float *dxall, float *dc, int M, int A, int P, void *stream);

/* PPO clipped surrogate gradient wrt the mean head (agent_ppo.py:58-65; rows with exps == 0 are excluded, :45);
 * inv_count = 1 / #selected rows; loss_acc (optional) accumulates the surrogate loss. */
int uhc_ppo_policy_grad(const float *mean, const float *log_std, const float *action, const float *adv, const float *fixed_logp, const float *exps,
                        float clip_eps, float inv_count, float *dmean, float *loss_acc, int M, int A, void *stream);
/* the same with 1 / #selected rows of the GLOBAL batch read from device memory (env-sharded multi-GPU update: the count arrives with the
 * gradient all-reduce, no host round trip) */
int uhc_ppo_policy_grad_dev(const float *mean, const float *log_std, const float *action, const float *adv, const float *fixed_logp, const float *exps,
                            float clip_eps, const float *inv_count_dev, float *dmean, float *loss_acc, int M, int A, void *stream);
/* value loss gradient (agent_pg.py:18-25): L = mean (v - returns)^2 ; _n: M_total = rows of the global batch (shard gradients then sum to the mean) */
int uhc_value_grad(const float *v, const float *ret, float *dv, float *loss_acc, int M, void *stream);
int uhc_value_grad_n(const float *v, const float *ret, float *dv, float *loss_acc, int M, long M_total, void *stream);
int uhc_sqsum(const float *x, long n, double *out_acc, void *stream);
/* torch.optim.Adam step (agent_copycat.py:160-177) with optional clip_grad_norm_ scale from *sqnorm (agent_ppo.py:53-56). */
int uhc_adam_step(float *p, const float *g, float *m, float *v, long n, float lr, float beta1, float beta2, float eps, int step,
                  const double *sqnorm_or_null, float max_norm, void *stream);

/* estimate_advantages (khrylib/rl/core/common.py:5-25) on a time-major [T][E] rollout; last_val = bootstrap V(s_T) or NULL (=0). */
int uhc_gae(const float *rew, const float *mask, const float *val, const float *last_val, float gamma, float tau, float *adv, float *ret, int T, int E,
            void *stream);
int uhc_normalize_advantages(float *adv, long n, double *scratch2, void *stream);   /* (A - mean) / std_unbiased, common.py:22 */
/* the two halves of it for a batch sharded over GPUs: local (sum, sum sq) -> [ride the gradient all-reduce] -> normalise with global moments / count */
int uhc_adv_moments(const float *adv, long n, double *out2, void *stream);
int uhc_adv_normalize(float *adv, long n, const double *mom2_dev, const double *ntotal_dev, void *stream);

/* ZFilter (khrylib/utils/zfilter.py:7-73): stats = [n, mean[D], S[D]] doubles; update!=0 merges the batch first (an empty batch, M = 0,
 * leaves the statistics as they are). y may be NULL. */
int uhc_zfilter(const float *x, float *y, int M, int D, double *stats, float clip, int update, void *stream);
/* the same with a caller-owned workspace of uhc_zfilter_workspace_doubles(D) doubles (needed inside a CUDA-graph capture: no allocation) */
int uhc_zfilter_ws(const float *x, float *y, int M, int D, double *stats, float clip, int update, double *workspace, void *stream);
int uhc_zfilter_workspace_doubles(int D);

#ifdef __cplusplus
}
#endif
#endif
