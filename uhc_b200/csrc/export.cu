// export.cu -- simulated qpos back to SMPL pose / translation on the device (include/uhc_export.h) and the evaluation's export kernel.
//
// Compiled on its own with -fmad=false (uhc_b200/build.py) like motion_lib.cu and eval.cu: smpl_export_core.h restates scipy's fp64
// arithmetic without contracted multiply-adds.  sm_90a.
#include <cuda_runtime.h>
#include <string>
#include <vector>
#include "../../include/uhc_eval.h"
#include "../../include/uhc_export.h"
#include "../../include/uhc_track.h"
#include "errors.h"
#include "eval_glue.h"
#include "sim_core.h"
#include "smpl_export_core.h"
#include "track_glue.h"

using namespace uhc;

namespace uhc {
namespace smplx {

// one thread per frame i < n
template <class Real>
__global__ void __launch_bounds__(128) k_qpos_to_smpl(const Real *__restrict__ qpos, long n, long pitch, const int *__restrict__ variant,
                                                      const double *__restrict__ body, double *__restrict__ pose, double *__restrict__ trans) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *root = body + (size_t)(variant ? variant[i] : 0) * MB * BODY6;
    double out[ROW];
    qpos_to_smpl<Real>(qpos + (size_t)i * pitch, root, out);
    for (int k = 0; k < POSE; k++) pose[(size_t)i * POSE + k] = out[k];
    for (int k = 0; k < 3; k++) trans[(size_t)i * 3 + k] = out[POSE + k];
}

cudaError_t launch_qpos_to_smpl(const void *qpos, int precision, long n, long pitch, const int *variant, const double *body,
                                double *pose, double *trans, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    if (precision == 32) k_qpos_to_smpl<float><<<blocks, 128, 0, st>>>((const float *)qpos, n, pitch, variant, body, pose, trans);
    else k_qpos_to_smpl<double><<<blocks, 128, 0, st>>>((const double *)qpos, n, pitch, variant, body, pose, trans);
    return cudaGetLastError();
}

// The evaluation's export (eval.cu, after k_eval_frame and before any fail_safe re-seat): every env i < n that recorded a frame in this step
// (its clips[i].frames grew past done[i], the count this kernel last saw) converts the state k_eval_frame just recorded into window row
// [i][slot].  Parked envs (i >= n) and envs that have stopped write nothing.
template <class Real>
__global__ void __launch_bounds__(128) k_eval_export(const Real *__restrict__ state, const int *__restrict__ istate, const int *__restrict__ clip_model,
                                                     const double *__restrict__ body, const UhcEvalClip *__restrict__ clips, int *__restrict__ done,
                                                     int n, int window, int slot, double *__restrict__ win_smpl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || slot >= window) return;
    const int frames = clips[i].frames;
    if (frames <= done[i]) return;
    done[i] = frames;
    const int v = clip_model ? clip_model[istate[(size_t)i * SI_SIZE + SI_CLIP]] : 0;
    qpos_to_smpl<Real>(state + (size_t)i * ST_SIZE + ST_Q, body + (size_t)v * MB * BODY6, win_smpl + ((size_t)i * window + slot) * ROW);
}

cudaError_t launch_eval_export(int precision, const void *state, const int *istate, const int *clip_model, const double *body, const UhcEvalClip *clips,
                               int *done, int n, int window, int slot, double *win_smpl, cudaStream_t st) {
    if (precision == 32)
        k_eval_export<float><<<(n + 127) / 128, 128, 0, st>>>((const float *)state, istate, clip_model, body, clips, done, n, window, slot, win_smpl);
    else
        k_eval_export<double><<<(n + 127) / 128, 128, 0, st>>>((const double *)state, istate, clip_model, body, clips, done, n, window, slot, win_smpl);
    return cudaGetLastError();
}

}  // namespace smplx
}  // namespace uhc

extern "C" {

int uhc_qpos_to_smpl(UhcEngine *e, const void *qpos_dev, int precision, long n, long qpos_pitch, const int *variant_dev_or_null,
                     double *pose_dev, double *trans_dev, void *stream) {
    if (!e) { uhc_err() = "uhc_qpos_to_smpl: null engine"; return -2; }
    if (n < 0) { uhc_err() = "uhc_qpos_to_smpl: n < 0"; return -2; }
    if (precision != 32 && precision != 64) { uhc_err() = "uhc_qpos_to_smpl: precision must be 32 or 64"; return -2; }
    if (qpos_pitch < 76) { uhc_err() = "uhc_qpos_to_smpl: qpos_pitch < 76"; return -2; }
    if (n > 0 && (!qpos_dev || !pose_dev || !trans_dev)) { uhc_err() = "uhc_qpos_to_smpl: null pointer"; return -2; }
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (variant_dev_or_null) {
        std::vector<int> v((size_t)n);
        cudaError_t ce = cudaMemcpyAsync(v.data(), variant_dev_or_null, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        if (ce != cudaSuccess) { uhc_err() = std::string("uhc_qpos_to_smpl: reading the variants: ") + cudaGetErrorString(ce); return -1; }
        const int ns = trackx::num_shapes(e);
        for (long i = 0; i < n; i++)
            if (v[(size_t)i] < 0 || v[(size_t)i] >= ns) { uhc_err() = "uhc_qpos_to_smpl: variant out of range"; return -2; }
    }
    const cudaError_t ce = smplx::launch_qpos_to_smpl(qpos_dev, precision, n, qpos_pitch, variant_dev_or_null, trackx::motion_model(e).body,
                                                      pose_dev, trans_dev, st);
    if (ce != cudaSuccess) { uhc_err() = std::string("uhc_qpos_to_smpl: ") + cudaGetErrorString(ce); return -1; }
    return 0;
}

int uhc_track_smpl(UhcEngine *e, const void *state_out_dev, double *pose_dev, double *trans_dev, void *stream) {
    if (!e || !state_out_dev || !pose_dev || !trans_dev) { uhc_err() = "uhc_track_smpl: null argument"; return -2; }
    evalx::EngineRefs R; evalx::engine_refs(e, &R);
    if (!trackx::tracking(e) || R.num_clips != R.E) { uhc_err() = "uhc_track_smpl: not tracking (uhc_track_begin), or the tracker's table was replaced"; return -2; }
    const cudaError_t ce = smplx::launch_qpos_to_smpl(state_out_dev, R.precision, R.E, UHC_TRACK_OUT, trackx::clip_models(e),
                                                      trackx::motion_model(e).body, pose_dev, trans_dev, (cudaStream_t)stream);
    if (ce != cudaSuccess) { uhc_err() = std::string("uhc_track_smpl: ") + cudaGetErrorString(ce); return -1; }
    return 0;
}

}  // extern "C"
