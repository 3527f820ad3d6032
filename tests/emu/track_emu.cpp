// track_emu.cpp -- TEST INFRASTRUCTURE: the tracker's per-env code compiled for the host (-DUHC_EMU, -ffp-contract=off): the stream's
// reset / push / rebase (uhc_b200/csrc/track_core.h) and the observation pass from the stored record (track_obs.h), next to the env
// step's emulation (emu.cpp, included whole so one library holds the env state both act on).
// Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#include "emu.cpp"
#include "../../uhc_b200/csrc/track_core.h"
#include "../../uhc_b200/csrc/track_obs.h"

extern "C" {
// one clip of T raw rows streamed into a window of H rows the way the tracker's kernels do it: reset with frames 0 and 1, one step
// (cur_t 0 -> 1), then per frame k = 2 .. T - 1 a push and a step.  Row t of the stream is read at window index cur_t + 1 right after
// the push that made it (out_next[t]) and at window index cur_t right before that push (out_cur[t - 1]); rows 0 and 1 are read after the
// reset.  Returns the number of rebases, or -1 if a push was dropped.
int emu_track_stream(int kind, int pose_dim, const double *rows, int T, int H, const int *parent, const int *ee, const double *body_f, int nshape,
                     int variant, double *out_next, double *out_cur) {
    using namespace uhc::motion;
    std::vector<double> body((size_t)nshape * MB * BODY6);
    motion_body_table(body_f, UHC_BODYF, nshape, body.data());
    MotionModel mm;
    motion_model_init(mm, parent, ee, body.data());
    const int row_w = kind == KIND_QPOS ? MQ : pose_dim + 3;
    std::vector<double> win((size_t)H * REC), raw(2 * (size_t)row_w);
    int have = 0, cur_t = 0, rebases = 0;
    track_reset_rows<double>(mm, kind, pose_dim, row_w, variant, rows, win.data(), raw.data(), &have);
    for (int k = 0; k < REC; k++) { out_next[k] = win[k]; out_next[REC + k] = win[REC + k]; out_cur[k] = win[k]; }
    cur_t = 1;
    for (int t = 2; t < T; t++) {
        for (int k = 0; k < REC; k++) out_cur[(size_t)(t - 1) * REC + k] = win[(size_t)cur_t * REC + k];
        const int h0 = have;
        if (!track_push_row<double>(mm, kind, pose_dim, row_w, variant, H, rows + (size_t)t * row_w, win.data(), raw.data(), &have, &cur_t)) return -1;
        if (have <= h0) rebases++;
        for (int k = 0; k < REC; k++) out_next[(size_t)t * REC + k] = win[(size_t)(cur_t + 1) * REC + k];
        cur_t += 1;
    }
    return rebases;
}

// the tracker's observation of env `env` from its stored record (track_obs.h), against row cur_t + 1 of its clip.  The work set is
// filled with NaN first, so nothing a previous step left in it can reach the observation
void emu_track_obs(void *h, int prec, int env, double *obs) {
    DISPATCH(h, prec, { std::memset((void *)&e->w, 0xFF, sizeof(e->w)); track_obs_warp<Real, double>(e->ev, env, e->w, obs); });
}
}
