// eval_emu.cpp -- TEST INFRASTRUCTURE: compiles the evaluation kernel's per-frame metric code (uhc_b200/csrc/eval_core.h) as host
// code (-DUHC_EMU, -ffp-contract=off) so it is checked against uhc_b200/metrics.py on a CPU-only box.
// Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#include "../../uhc_b200/csrc/eval_core.h"

using namespace uhc;

extern "C" {
// the per-frame values of one episode of T frames, frame by frame through the kernel's code: out = [T][6]
// (mpjpe_g, mpjpe, pa_mpjpe, vel (0 at frame 0), accel (0 at frames 0, 1), |I - X_pred X_gt^-1|_F)
void emu_eval_frames(int T, const double *qpos_pred, const double *qpos_gt, const double *jpos_pred, const double *jpos_gt, double *out) {
    for (int k = 0; k < T; k++) {
        const double *pj1 = k >= 1 ? jpos_pred + (k - 1) * 72 : nullptr, *gj1 = k >= 1 ? jpos_gt + (k - 1) * 72 : nullptr;
        const double *pj2 = k >= 2 ? jpos_pred + (k - 2) * 72 : nullptr, *gj2 = k >= 2 ? jpos_gt + (k - 2) * 72 : nullptr;
        evalm::eval_frame(qpos_pred + k * 76, qpos_gt + k * 76, jpos_pred + k * 72, jpos_gt + k * 72, pj1, gj1, pj2, gj2, out + k * evalm::EV_N);
    }
}
}
