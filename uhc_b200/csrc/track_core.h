// track_core.h -- the per-env logic of the tracker's target stream (track.cu): rows of a window of H expert-table records built one raw
// frame at a time with motion_core.h's motion_frame, and the rebase that keeps the window from running out.  Shared with the host
// emulation (tests/emu, -DUHC_EMU, -ffp-contract=off) like motion_core.h.
//
// A stream's row k is the record of the raw pair (k - 1, k) (row 0: the pair (0, 1)), which is exactly what motion_frame computes for
// row k of the whole clip: a streamed clip equals the same clip loaded with uhc_load_motions, bit for bit.  The raw frame of the last
// pushed row is kept in fp64 per env (raw[0]); the new frame lands in raw[1] and the pair is read as a 2-row clip at t = 1.
#pragma once
#include "motion_core.h"

namespace uhc {
namespace motion {

// frames f01 = [2][row_w] become rows 0 and 1 of the window; raw[0] <- frame 1; *have = 2
template <class Out>
UHC_MDEV void track_reset_rows(const MotionModel &m, int kind, int pose_dim, int row_w, int variant, const double *f01, Out *rows, double *raw,
                               int *have) {
    motion_frame<Out>(m, kind, pose_dim, f01, row_w, 0, variant, rows);
    motion_frame<Out>(m, kind, pose_dim, f01, row_w, 1, variant, rows + REC);
    for (int i = 0; i < row_w; i++) raw[i] = f01[row_w + i];
    *have = 2;
}

// appends `frame` as row *have of the window [H][REC].  A full window first moves rows cur_t .. have - 1 (the ones a step can still read:
// cur_t for the fail_safe re-seat, cur_t + 1 .. for the targets) to the front and lowers cur_t and have by the same offset.  Returns 1,
// or 0 when the window holds no row it may drop (cur_t = 0: the caller pushed H - 1 frames ahead of its steps) and the frame is dropped.
template <class Out>
UHC_MDEV int track_push_row(const MotionModel &m, int kind, int pose_dim, int row_w, int variant, int H, const double *frame, Out *rows,
                            double *raw, int *have, int *cur_t) {
    if (*have >= H) {
        const int off = *cur_t;
        if (off <= 0) return 0;
        for (int r = off; r < *have; r++)
            for (int k = 0; k < REC; k++) rows[(size_t)(r - off) * REC + k] = rows[(size_t)r * REC + k];
        *have -= off; *cur_t -= off;
    }
    for (int i = 0; i < row_w; i++) raw[row_w + i] = frame[i];
    motion_frame<Out>(m, kind, pose_dim, raw, row_w, 1, variant, rows + (size_t)(*have) * REC);
    for (int i = 0; i < row_w; i++) raw[i] = raw[row_w + i];
    *have += 1;
    return 1;
}

}  // namespace motion
}  // namespace uhc
