"""GPU: the phase cycle accounting of k_env_step (-DUHC_PHASE_CLOCKS, scripts/step_phase_cycles.py) only reads clocks.  The instrumented library,
with the accounting switched on, runs a few hundred rollout steps of the bench's default configuration to the same bits as the production
library: every step's observations, rewards and masks, and the env state records at the end."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E, T, NPHASE = 4096, 300, 13      # the bench's env count: two full waves of 16-warp CTAs

CHILD = r"""
import ctypes as C, hashlib, json, sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
from bench import make_clip
from uhc_b200.agent import BatchedAgent, RolloutBuffer
E, T, clocks, out = %(E)d, %(T)d, %(clocks)d, %(out)r
ex, shape = make_clip()
agent = BatchedAgent(E, [ex], [shape], device=0, seed=1)
agent.reset_envs()
cyc = torch.zeros(E * %(nphase)d + 64, dtype=torch.int64, device=agent.dev)   # [E][NPHASE] and a guard
nphase = agent.engine.lib.uhc_phase_clocks(agent.engine.h, C.c_void_p(cyc.data_ptr())) if clocks else 0
buf = RolloutBuffer(1, E, agent.dev, agent.act_dim, agent.obs_dim)
h = hashlib.sha256()
for t in range(T):
    agent.rollout(buf, 1, 0)
    for x in (agent.obs, buf.actions[0], buf.rewards[0], buf.masks[0], buf.fails[0]):
        h.update(x.cpu().numpy().tobytes())
st = agent.engine.get_states()
np.savez(out, **{k: np.asarray(v) for k, v in st.items()}, digest=np.frombuffer(h.digest(), np.uint8),
         counters=np.array(json.dumps(agent.engine.counters)), nphase=nphase, cycles=cyc.cpu().numpy())
"""


def _run(so, clocks, out):
    env = dict(os.environ, UHC_B200_SO=so)
    code = CHILD % dict(root=ROOT, E=E, T=T, clocks=clocks, out=out, nphase=NPHASE)
    subprocess.run([sys.executable, "-c", code], env=env, check=True, cwd=ROOT)
    return np.load(out)


def test_instrumented_build_steps_to_the_same_bits(tmp_path):
    from uhc_b200 import build
    so = build.build(so=str(tmp_path / "libuhc_b200.so"), defines=["UHC_PHASE_CLOCKS"])
    prod = _run(build.build(), 0, str(tmp_path / "prod.npz"))
    inst = _run(so, 1, str(tmp_path / "inst.npz"))
    assert int(inst["nphase"]) == NPHASE
    cyc = inst["cycles"][:E * NPHASE].reshape(E, NPHASE)
    assert (cyc >= 0).all() and (cyc.sum(1) > 0).all(), "every env's warp accounts its cycles"
    assert not inst["cycles"][E * NPHASE:].any(), "nothing is written past the E x NPHASE buffer"
    assert np.array_equal(prod["digest"], inst["digest"]), "per-step outputs differ between the production and the instrumented build"
    for k in ("qpos", "qvel", "xpos", "bquat", "cur_t", "clip", "start", "len", "episode", "flags", "newton_iters", "ncon"):
        assert np.array_equal(prod[k], inst[k]), k
    assert str(prod["counters"]) == str(inst["counters"])
