// group_core.h -- row-tile schedule of the grouped tensor-core GEMM (k_linear_tc_grouped, mlp_wgmma.cu).
//
// G groups of rows, group g = rows [row0[g], row0[g] + rows[g]) of the activations, each multiplied by its own weights.  Every group is cut
// into 128-row tiles that start at the group's first row, so a tile never holds rows of two groups' products: the tile reads its group's
// weights and its stores stop at the group's last row.  Rows between or after the groups are never written.  tile0[g] is the first
// tile of group g and tile0[G] the number of tiles, at most ceil(sum rows / 128) + G - 1 (per 128-column block of the output).
// Written like eval_core.h: the same source compiles as CUDA code and, with -DUHC_EMU, as host code for the CPU tests.
#pragma once

#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_GHD __host__ __device__ __forceinline__
#else
#define UHC_GHD static inline
#endif

namespace uhc {
namespace grp {

constexpr int MAX_GROUPS = 64, TILE_ROWS = 128;

struct TilePlan {
    int G, pad;
    int row0[MAX_GROUPS], rows[MAX_GROUPS], tile0[MAX_GROUPS + 1];
};

// validates the groups (1 <= G <= MAX_GROUPS, rows >= 1, ascending and disjoint, inside [0, M)) and fills the plan; 0, or -2 on a bad argument
UHC_GHD int plan_tiles(int G, const int *row0, const int *rows, int M, TilePlan *p) {
    if (G < 1 || G > MAX_GROUPS || !row0 || !rows) return -2;
    p->G = G; p->pad = 0; p->tile0[0] = 0;
    for (int g = 0; g < G; g++) {
        if (rows[g] < 1 || row0[g] < 0 || row0[g] > M - rows[g]) return -2;
        if (g > 0 && row0[g] < row0[g - 1] + rows[g - 1]) return -2;
        p->row0[g] = row0[g]; p->rows[g] = rows[g];
        p->tile0[g + 1] = p->tile0[g] + (rows[g] + TILE_ROWS - 1) / TILE_ROWS;
    }
    return 0;
}

// the group of row tile t (0 <= t < tile0[G]): the last g with tile0[g] <= t
UHC_GHD int tile_group(const TilePlan &p, int t) {
    int lo = 0, hi = p.G - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (p.tile0[mid] <= t) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// rows [*first, *end) of tile t; the tile's loads start at *first, its stores stop before *end
UHC_GHD int tile_rows(const TilePlan &p, int t, int *first, int *end) {
    const int g = tile_group(p, t);
    *first = p.row0[g] + (t - p.tile0[g]) * TILE_ROWS;
    *end = p.row0[g] + p.rows[g];
    return g;
}

}  // namespace grp
}  // namespace uhc
