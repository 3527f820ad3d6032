// export_emu.cpp -- TEST INFRASTRUCTURE: compiles the device SMPL export's per-frame code (uhc_b200/csrc/smpl_export_core.h) as host code
// (-DUHC_EMU, -ffp-contract=off) so the kernel math is checked against the reference's qpos_to_smpl on a CPU-only box.
// Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../uhc_b200/csrc/smpl_export_core.h"

using namespace uhc;

extern "C" {
// n frames of qpos (row pitch `pitch` doubles) -> out [n][75] (pose 72, trans 3); body_f = [nshape][24][20] of the shape variants,
// variant = per frame (NULL = variant 0)
void emu_qpos_to_smpl(long n, const double *qpos, long pitch, const double *body_f, int nshape, const int *variant, double *out) {
    std::vector<double> body((size_t)nshape * motion::MB * motion::BODY6);
    motion::motion_body_table(body_f, UHC_BODYF, nshape, body.data());
    for (long i = 0; i < n; i++)
        smplx::qpos_to_smpl<double>(qpos + (size_t)i * pitch, body.data() + (size_t)(variant ? variant[i] : 0) * motion::MB * motion::BODY6,
                                    out + (size_t)i * smplx::ROW);
}
}
