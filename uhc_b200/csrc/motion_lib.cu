// motion_lib.cu -- the device motion library: expert-table records built from raw SMPL / qpos rows (motion_core.h), one thread per
// frame.  Compiled on its own with -fmad=false (uhc_b200/build.py): the records restate motion_lib.py's fp64 arithmetic without
// contracted multiply-adds, so they agree with the host-built table to the rounding of the math library.  sm_90a.
// The C ABI (uhc_load_motions, uhc_get_clip_frames) is in step_kernel.cu, next to uhc_load_clips whose contract it shares.
#include <cuda_runtime.h>
#include "motion_core.h"

namespace uhc {
namespace motion {

template <class Out>
__global__ void __launch_bounds__(128) k_motion_frames(MotionModel m, int kind, int pose_dim, const double *__restrict__ rows,
                                                      const int *__restrict__ clip_adr, const int *__restrict__ fk_model, int c0, int c1, int nf,
                                                      Out *__restrict__ table) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    const int f0 = clip_adr[c0], f = f0 + i;
    int lo = c0, hi = c1 - 1;          // clip of frame f: the last clip starting at or before it
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (clip_adr[mid] <= f) lo = mid; else hi = mid - 1; }
    const int row_w = kind == KIND_QPOS ? MQ : pose_dim + 3;
    motion_frame<Out>(m, kind, pose_dim, rows + (size_t)(clip_adr[lo] - f0) * row_w, row_w, f - clip_adr[lo], fk_model ? fk_model[lo] : 0,
                      table + (size_t)f * REC);
}

template <class Out>
cudaError_t launch_motion_frames(const MotionModel &m, int kind, int pose_dim, const double *rows, const int *clip_adr, const int *fk_model,
                                 int c0, int c1, int nf, Out *table, cudaStream_t st) {
    if (nf <= 0) return cudaSuccess;
    k_motion_frames<Out><<<(nf + 127) / 128, 128, 0, st>>>(m, kind, pose_dim, rows, clip_adr, fk_model, c0, c1, nf, table);
    return cudaGetLastError();
}
template cudaError_t launch_motion_frames<float>(const MotionModel &, int, int, const double *, const int *, const int *, int, int, int, float *, cudaStream_t);
template cudaError_t launch_motion_frames<double>(const MotionModel &, int, int, const double *, const int *, const int *, int, int, int, double *, cudaStream_t);

}  // namespace motion
}  // namespace uhc
