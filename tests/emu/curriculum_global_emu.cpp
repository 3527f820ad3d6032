// curriculum_global_emu.cpp -- TEST INFRASTRUCTURE: compiles the global curriculum's payload rules (uhc_b200/csrc/curriculum_core.h:
// stage_entry, unpack_entry, stage_exact) as host code (-DUHC_EMU, -ffp-contract=off), in the steps k_cur_stage / k_cur_unpack take, so the
// stage -> sum -> unpack round trip is checked on a CPU-only box.  Never loaded by the product path.
#define UHC_EMU 1
#include <math.h>
#include "../../uhc_b200/csrc/curriculum_core.h"

using namespace uhc::cur;

extern "C" {
// n log entries -> out [n][3] as k_cur_stage writes them
void emu_cur_stage(int n, const int *clip_log, const float *pct_log, const int *start_log, float *out) {
    for (int i = 0; i < n; i++) stage_entry(clip_log[i], pct_log[i], start_log[i], out + 3 * (size_t)i);
}
// a summed payload [n][3] back into the three logs, as k_cur_unpack reads it
void emu_cur_unpack(int n, const float *in, int *clip_log, float *pct_log, int *start_log) {
    for (int i = 0; i < n; i++) unpack_entry(in + 3 * (size_t)i, clip_log + i, pct_log + i, start_log + i);
}
int emu_cur_stage_exact(long long num_clips, long long longest_clip) { return stage_exact(num_clips, longest_clip) ? 1 : 0; }
}
