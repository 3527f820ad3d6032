// curriculum_emu.cpp -- TEST INFRASTRUCTURE: compiles the device curriculum's rules (uhc_b200/csrc/curriculum_core.h) as host code
// (-DUHC_EMU, -ffp-contract=off), in the steps curriculum.cu takes, so they are checked against the reference's Python on a CPU-only box.
// Never loaded by the product path.
#define UHC_EMU 1
#include <math.h>
#include <vector>
#include "../../uhc_b200/csrc/curriculum_core.h"

using namespace uhc::cur;

extern "C" {
// one rollout's [N] log into the rings: per clip count, rank in log order, keep the last M at (head + rank) mod M, advance
void emu_cur_append(int C, int M, int *meta, float *pct, int *start, int N, const int *clip_log, const float *pct_log, const int *start_log) {
    std::vector<int> n(C, 0), rank(N, 0);
    for (int i = 0; i < N; i++) if (clip_log[i] >= 0 && clip_log[i] < C) rank[i] = n[clip_log[i]]++;
    for (int i = 0; i < N; i++) {
        const int c = clip_log[i];
        if (c < 0 || c >= C || !keep_rank(rank[i], n[c], M)) continue;
        const int slot = rank_slot(meta, M, c, rank[i] % M);
        pct[(size_t)c * M + slot] = pct_log[i]; start[(size_t)c * M + slot] = start_log[i];
    }
    for (int c = 0; c < C; c++) ring_advance(meta, M, c, n[c]);
}
// the weights (w [C], fp32) and the CDF as k_cur_weights computes them (any history; else the sample_keys rule)
void emu_cur_weights(int C, int M, const int *meta, const float *pct, double temp, double freq, int t_max, const int *clip_len, float *w, float *cdf) {
    std::vector<double> p(C);
    int any = 0;
    for (int c = 0; c < C; c++) { any |= meta[2 * c + 1] > 0; p[c] = exp(-success_ewma(pct, meta, M, c) / temp); }
    const double sum = pairwise_sum(p.data(), C);
    double acc = 0.0;
    for (int c = 0; c < C; c++) {
        w[c] = any ? clip_weight(p[c], sum, freq, C) : (float)(t_max > 0 ? clip_len[c] / t_max + 1 : 1);
        acc += (double)w[c]; cdf[c] = (float)acc;
    }
}
double emu_pairwise_sum(const double *a, int n) { return pairwise_sum(a, n); }
// the exact law of a re-seed's start frame for clip c of length L
void emu_cur_start_law(int M, const int *meta, const float *pct, const int *start, int c, int L, int t_min, double prec_freq, double *pmf) {
    start_law(pct, start, meta, M, c, L, t_min, prec_freq, pmf);
}
// the sampler's draw from explicit uniforms (what the kernel does with its hash)
int emu_cur_draw_start(int M, const int *meta, const float *pct, const int *start, int c, int L, int t_min, float prec_freq, float u_coin, float u_pick, float u_start) {
    return draw_start(pct, start, meta, M, c, L, t_min, prec_freq, u_coin, u_pick, u_start);
}
}
