// subject_emu.cpp -- TEST INFRASTRUCTURE: compiles the subject body builder's per-item code (uhc_b200/csrc/subject_core.h) as host code
// (-DUHC_EMU, -ffp-contract=off) and runs one subject's items in the order k_subject runs them, so the kernel math is checked against
// tests/subject_ref.py on a CPU-only box.  Never loaded by the product path (uhc_b200/subject_body.py only loads the CUDA library).
#define UHC_EMU 1
#include "../../uhc_b200/csrc/subject_core.h"

using namespace uhc::subj;

extern "C" {
// one subject: map_basis [24][11][12] and off_basis [24][11][3] of its gender, beta [10]; base tables as UhcModelHost holds them (variant 0);
// writes body_f [24][20], hull [nvert][3], maps [24][12].  Returns 0, or 1 + the first body whose map has det A <= 0.
int emu_subject_body(const double *map_basis, const double *off_basis, const double *beta, const double *bf0, const double *hull0, int nvert,
                     const int *hull_adr, const int *hull_num, const int *parent, const int *sub_end, const double *dof_f, double *body_f,
                     double *hull, double *maps) {
    static double bf[NB][BODYF], L[NTRI], part[NB * 3];
    static Rest R;
    double arm[NV];
    for (int i = 0; i < NV; i++) arm[i] = dof_f[4 * i];
    for (int b = 0; b < NB; b++) {
        eval_map(map_basis + b * NTERM * MAPW, beta, maps + b * MAPW);
        if (!(det3(maps + b * MAPW) > 0.0)) return b + 1;
        eval_offset(off_basis + b * NTERM * 3, beta, bf0 + b * BODYF, bf[b]);
        mass_props(maps + b * MAPW, bf0 + b * BODYF, bf[b]);
        bf[b][18] = bf0[b * BODYF + 18]; bf[b][19] = bf0[b * BODYF + 19];
    }
    for (int b = 0; b < NB; b++)
        for (int k = 0; k < hull_num[b]; k++) {
            const int v = hull_adr[b] + k;
            apply(maps + b * MAPW, hull0 + 3 * v, hull + 3 * v);
        }
    for (int b = 0; b < NB; b++) {
        for (int c = 0; c < 3; c++) {
            R.gpos[b][c] = b == 0 ? bf[0][c] : R.gpos[parent[b]][c] + bf[b][c];
            R.xipos[b][c] = R.gpos[b][c] + bf[b][3 + c];
        }
        R.mass[b] = bf[b][6];
        for (int k = 0; k < 6; k++) R.inertia[b][k] = bf[b][7 + k];
        R.parent[b] = parent[b];
        R.sub_end[b] = sub_end[b];
    }
    for (int i = 0; i < NV; i++)
        for (int j = 0; j <= i; j++) L[tri(i, j)] = m_entry(R, arm, i, j);
    for (int k = 0; k < NV; k++) {
        chol_pivot(L, k);
        for (int i = k + 1; i < NV; i++) chol_col(L, k, i);
        for (int i = k + 1; i < NV; i++)
            for (int j = k + 1; j <= i; j++) chol_update(L, k, i, j);
    }
    double y[NV];
    for (int q = 0; q < NB * 3; q++) part[q] = invw_part(R, L, q / 3, q % 3, y);
    for (int b = 0; b < NB; b++) bf[b][13] = (part[3 * b] + part[3 * b + 1] + part[3 * b + 2]) / 3.0;
    for (int b = 0; b < NB; b++) {
        for (int c = 0; c < BODYF; c++) body_f[b * BODYF + c] = bf[b][c];
        double sp[4] = {0.0, 0.0, 0.0, 0.0};
        if (hull_num[b] > 0) sphere(hull + 3 * hull_adr[b], hull_num[b], sp);
        for (int c = 0; c < 4; c++) body_f[b * BODYF + 14 + c] = sp[c];
    }
    (void)nvert;
    return 0;
}
}
