// group_emu.cpp -- TEST INFRASTRUCTURE: compiles the grouped GEMM's row-tile schedule (uhc_b200/csrc/group_core.h) as host code so the
// CPU tests can check it.  Never loaded by the product path.
#define UHC_EMU 1
#include "../../uhc_b200/csrc/group_core.h"

using namespace uhc;

extern "C" {
// the plan of G groups over M rows: returns plan_tiles' code; on success tiles = tile count, and per tile t: group[t], first[t], end[t]
// (the caller sizes the outputs for max_tiles tiles; -3 if the plan has more)
int emu_group_tiles(int G, const int *row0, const int *rows, int M, int max_tiles, int *tiles, int *group, int *first, int *end) {
    grp::TilePlan p;
    const int rc = grp::plan_tiles(G, row0, rows, M, &p);
    if (rc) return rc;
    *tiles = p.tile0[G];
    if (*tiles > max_tiles) return -3;
    for (int t = 0; t < *tiles; t++) group[t] = grp::tile_rows(p, t, first + t, end + t);
    return 0;
}
}
