// motion_emu.cpp -- TEST INFRASTRUCTURE: compiles the device motion library's per-frame code (uhc_b200/csrc/motion_core.h) as host
// code (-DUHC_EMU, -ffp-contract=off) so every line of the kernel math is checked against uhc_b200/motion_lib.py on a CPU-only box.
// Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../uhc_b200/csrc/motion_core.h"

using namespace uhc;

extern "C" {
// expert table [sum(len)][576] of nclips clips from raw rows, frame by frame through the motion kernel's code;
// body_f = [nshape][24][20] of the shape variants, fk_model = variant per clip (NULL = variant 0)
void emu_motion_table(int nclips, const int *len, int kind, int pose_dim, const double *rows, const int *parent, const int *ee,
                      const double *body_f, int nshape, const int *fk_model, double *out) {
    std::vector<double> body((size_t)nshape * motion::MB * motion::BODY6);
    motion::motion_body_table(body_f, UHC_BODYF, nshape, body.data());
    motion::MotionModel mm;
    motion::motion_model_init(mm, parent, ee, body.data());
    const int row_w = kind == motion::KIND_QPOS ? motion::MQ : pose_dim + 3;
    size_t f0 = 0;
    for (int c = 0; c < nclips; c++) {
        for (int t = 0; t < len[c]; t++)
            motion::motion_frame<double>(mm, kind, pose_dim, rows + f0 * row_w, row_w, t, fk_model ? fk_model[c] : 0, out + (f0 + t) * motion::REC);
        f0 += len[c];
    }
}
}
