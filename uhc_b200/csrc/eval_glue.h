// eval_glue.h -- internal interface of the device evaluation (eval.cu) and the tracker (track.cu) to the engine (step_kernel.cu) and to
// the policy forward of the rollout (rollout.cu).  Not part of the C ABI.  Host-only declarations and plain structs.
#pragma once
#include <cuda_runtime.h>
#include <string>
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../include/uhc_rollout.h"

namespace uhc {
namespace evalx {

// the engine's device state and its host-API staging buffers (obs / action / step outputs, E rows each)
struct EngineRefs {
    int E, precision, obs_dim, act_dim, num_clips;
    void *state; int *istate; const void *expert; const int *clip_adr;
    const int *clip_len_h;    // host copy of the clip lengths
    unsigned long long view_gen;   // changes with every cfg / clip-table / clip-model / CDF / neutral-pose update (graphs hold those by value)
    float *obs, *act, *rew, *cinfo, *pct; int *fail, *end;
};
void engine_refs(UhcEngine *e, EngineRefs *out);                                            // step_kernel.cu
// fail_safe re-seat of every env i < n with reseat[i] != 0: uhc_env_set_state_batch's reset-with-override onto the expert qpos / qvel
// of frame min(cur_t, len - 1), rounded to fp32, keeping cur_t and the body quaternions; one launch, no host work
cudaError_t launch_reseat(UhcEngine *e, int n, const int *reseat, cudaStream_t st);       // step_kernel.cu
// changes whenever the sampler's curriculum view (rings, fit_clip, prec_freq, CDF pointer under the curriculum) changes; the rollout's
// graphs are keyed on it                                                                                                   // step_kernel.cu
unsigned long long curriculum_gen(const UhcEngine *e);
// the policy of a rollout as a flat net list: one MLP (PolicyGaussian, nprim = 0: nets[0]) or a PolicyMCP mixture (nets[0 .. nprim-1] =
// primitives, nets[nprim] = composer).  Zeroed before it is filled, so its bytes can go into a graph key
struct Policy { int nprim; int pad; UhcMlp nets[UHC_MCP_MAX_PRIM + 1]; };
// The four calls below return 0 or an error code with its text in uhc_err() (errors.h).
// policy of an evaluation or a tracker step: converts and validates it (-2) and sizes the rollout's policy scratch outside any capture;
// *gen changes whenever that scratch is reallocated (graphs holding the old pointers must be dropped)
int policy_prepare(UhcEngine *e, const UhcMlp *mlp, const UhcMcp *mcp, Policy *pol, unsigned long long *gen);   // rollout.cu
// obs -> ZFilter (no update) -> policy -> action (the mean where mean_action[e] != 0); enqueues only (capturable)
int policy_enqueue(UhcEngine *e, const Policy &pol, const float *obs, const float *log_std, double *zstats, float zclip,
                   const unsigned char *mean_action, float *action, cudaStream_t st);                 // rollout.cu
// the grouped evaluation (uhc_eval_run_groups): G policies (mlps[G] or mcps[G]) of one architecture, group g on rows [row0[g], row0[g + 1]).
// groups_prepare converts and validates them (-2) and sizes the grouped policy scratch, a second instance (never the rollout's own); *gen
// changes whenever that scratch is reallocated.  groups_enqueue: obs -> ZFilter of each group (zstats[g], no update) -> grouped GEMMs
// (+ mixture head) -> the mean action (with mean_action all ones) of rows 0 .. row0[G] - 1; enqueues only (capturable).
int groups_prepare(UhcEngine *e, int G, const UhcMlp *mlps, const UhcMcp *mcps, std::vector<Policy> *pols, unsigned long long *gen);   // rollout.cu
int groups_enqueue(UhcEngine *e, const std::vector<Policy> &pols, const int *row0, const double *const *zstats, float zclip, const float *obs,
                   const unsigned char *mean_action, float *action, cudaStream_t st);                 // rollout.cu

}  // namespace evalx
}  // namespace uhc
