// fwd_emu.cpp -- TEST INFRASTRUCTURE: the smooth phase's forward pass of sim_core.h (kin_rne_forward, project_force, collide) compiled as the
// host lane-loop emulation (-DUHC_EMU), with everything it writes into the work set handed back, so that its bits can be pinned on a CPU.
// Never loaded by the product path.
#include "emu.cpp"

// One fp32 forward pass on (qpos, qvel).  The work set is zeroed first, so slots a pass leaves alone read 0.
//   fout: xpos 72 | xmat 216 | xipos 72 | S 75*6 | Vb 144 | Ab 144 | Ib 240 | Fb 144 | C 75 | cdist 40 | cr 120  (FWD_NF floats)
//   iout: cbody 40 | bcon_adr 25 | ncon | upper_contact | con_overflow                                           (FWD_NI ints)
extern "C" void emu_fwd_pass(void *h, const double *qpos, const double *qvel, float *fout, int *iout) {
    Emu<float> *e = (Emu<float> *)h;
    Work<float> &w = e->w;
    std::memset((void *)&w, 0, sizeof(w));
    for (int i = 0; i < NQ; i++) w.q[i] = (float)qpos[i];
    for (int i = 0; i < NV; i++) w.v[i] = (float)qvel[i];
    const Model<float> &m = e->ev.model;
    TOPO_DECL(m);
    kin_rne_forward(m, w, tp);
    project_force(m, w, w.Fb, w.C, 1.0f, (const float *)nullptr);
    collide(m, w, tp);
    float *f = fout;
    auto put = [&f](const float *src, int n) { std::memcpy(f, src, n * sizeof(float)); f += n; };
    put(&w.xpos[0][0], NB * 3); put(&w.xmat[0][0], NB * 9); put(&w.xipos[0][0], NB * 3); put(&w.S[0][0], NV * 6);
    put(&w.Vb[0][0], NB * 6); put(&w.Ab[0][0], NB * 6); put(&w.Ib[0][0], NB * 10); put(&w.Fb[0][0], NB * 6); put(w.C, NV);
    put(w.cdist, MAXCON); put(&w.cr[0][0], MAXCON * 3);
    int *o = iout;
    std::memcpy(o, w.cbody, MAXCON * sizeof(int)); o += MAXCON;
    std::memcpy(o, w.bcon_adr, (NB + 1) * sizeof(int)); o += NB + 1;
    o[0] = w.ncon; o[1] = w.upper_contact; o[2] = w.con_overflow;
}
