// floor_emu.cpp -- TEST INFRASTRUCTURE: compiles the floor measurements' per-frame code (uhc_b200/csrc/floor_core.h) as host code
// (-DUHC_EMU, -ffp-contract=off), one frame as one warp computes it, so the kernel math and its reduction order are checked against
// tests/floor_ref.py on a CPU-only box.  Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#include <vector>
#include "../../include/uhc_b200.h"
#include "../../uhc_b200/csrc/floor_core.h"

using namespace uhc;

namespace {
struct Model {
    std::vector<double> body; std::vector<unsigned char> vbody; motion::MotionModel mm; const double *hull; int nvert;
    Model(const int *parent, const int *ee, const double *body_f, int nshape, const double *hull_, int nvert_, const int *hull_adr, const int *hull_num)
        : body((size_t)nshape * motion::MB * motion::BODY6), vbody((size_t)nvert_), hull(hull_), nvert(nvert_) {
        motion::motion_body_table(body_f, UHC_BODYF, nshape, body.data());
        motion::motion_model_init(mm, parent, ee, body.data());
        for (int b = 0; b < motion::MB; b++) for (int k = 0; k < hull_num[b]; k++) vbody[(size_t)hull_adr[b] + k] = (unsigned char)b;
    }
    floorm::Hull variant_hull(int v) const { return floorm::Hull{hull + (size_t)v * nvert * 3, vbody.data(), nvert}; }
    const double *variant_body(int v) const { return body.data() + (size_t)v * motion::MB * motion::BODY6; }
};
}  // namespace

extern "C" {
// uhc_floor_qpos: n rows of qpos at `pitch` doubles, variant / first per row or NULL; out = [n][5]
void emu_floor_qpos(long n, const double *qpos, long pitch, const int *variant, const int *first, const int *parent, const int *ee, const double *body_f,
                    int nshape, const double *hull, int nvert, const int *hull_adr, const int *hull_num, double *out) {
    const Model M(parent, ee, body_f, nshape, hull, nvert, hull_adr, hull_num);
    for (long i = 0; i < n; i++) {
        const int v = variant ? variant[i] : 0;
        const bool has_prev = i > 0 && !(first && first[i]);
        floorm::frame_rows(M.mm, M.variant_hull(v), M.variant_body(v), qpos + i * pitch, has_prev ? qpos + (i - 1) * pitch : nullptr, out + i * floorm::NCOL,
                           nullptr);
    }
}
// uhc_motion_floor: raw rows of nclips clips; out = [sum(len)][5], feet = [sum(len)][4]
void emu_motion_floor(int nclips, const int *len, int kind, int pose_dim, const double *rows, const int *fk_model, const int *parent, const int *ee,
                      const double *body_f, int nshape, const double *hull, int nvert, const int *hull_adr, const int *hull_num, double *out, double *feet) {
    const Model M(parent, ee, body_f, nshape, hull, nvert, hull_adr, hull_num);
    const int row_w = kind == motion::KIND_QPOS ? motion::MQ : pose_dim + 3;
    size_t f = 0;
    for (int c = 0; c < nclips; c++) {
        const int v = fk_model ? fk_model[c] : 0;
        double q[2][motion::MQ];
        for (int t = 0; t < len[c]; t++, f++) {
            motion::m_load_qpos(M.mm, kind, pose_dim, rows + f * row_w, M.variant_body(v), q[t & 1]);
            floorm::frame_rows(M.mm, M.variant_hull(v), M.variant_body(v), q[t & 1], t > 0 ? q[(t - 1) & 1] : nullptr, out + f * floorm::NCOL,
                               feet + f * floorm::NFEET);
        }
    }
}
}
