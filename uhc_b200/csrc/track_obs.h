// track_obs.h -- the tracker's observation pass, one warp per env: the observation of the env's STORED state against row cur_t + 1,
// through the step kernel's own write_obs.  Shared by the CUDA kernel (step_kernel.cu k_track_obs) and the host emulation (tests/emu).
//
// The step kernel writes its observation at the end of a step from the work set: q / v after the last integration, xpos / xipos of the
// last forward pass, xquat of world_quat.  store_state then writes exactly those arrays into the record (ST_Q, ST_V, ST_XPOS, ST_XIPOS,
// ST_XQUAT), so loading them back and calling write_obs again reproduces that observation.  The reset path stores the same arrays.
#pragma once
#include "env_step.h"

namespace uhc {

template <class Real, class ObsT>
UHC_DEV void track_obs_warp(const EngineView<Real> &ev, int env, Work<Real> &w, ObsT *obs) {
    const int *is = ev.istate + (size_t)env * SI_SIZE;
    const Real *st = ev.state + (size_t)env * ST_SIZE;
    LANES_BEGIN
    for (int i = lane; i < NQ; i += 32) w.q[i] = st[ST_Q + i];
    for (int i = lane; i < NV; i += 32) w.v[i] = st[ST_V + i];
    for (int i = lane; i < 72; i += 32) { (&w.xpos[0][0])[i] = st[ST_XPOS + i]; (&w.xipos[0][0])[i] = st[ST_XIPOS + i]; }
    for (int i = lane; i < 96; i += 32) (&w.xquat[0][0])[i] = st[ST_XQUAT + i];
    if (lane == 0) w.cfg = ev.cfg;
    LANES_END
    write_obs(ev, w, is[SI_CLIP], is[SI_START], is[SI_LEN], is[SI_CUR_T] + 1, obs);
}

}  // namespace uhc
