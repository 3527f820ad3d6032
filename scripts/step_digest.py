#!/usr/bin/env python
"""step_digest.py -- a digest of what the bench's rollout computes, to check that a change to k_env_step keeps every bit.

  python scripts/step_digest.py --out FILE.json [--so LIB] [--envs 4096] [--steps 300]

Runs the bench's rollout (its clip, agent and seed; 4096 envs, two full waves of 16-warp CTAs) for --steps control steps on the library
--so names (default: the production library the package loads) in a child process, and writes one JSON object:

  outputs_sha256  SHA-256 over every step's next observations, actions, rewards, masks and fail flags, in step order
  state_sha256    SHA-256 of each array of the env state records at the end (qpos, qvel, xpos, bquat and the integer record)
  counters        the engine's device counters at the end

tests/golden/step_digest.json was written by this script on an H100 from the library before k_env_step's code was made smaller;
tests/test_gpu_step_footprint.py compares every later build with it.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "step_digest.json")

CHILD = r"""
import hashlib, json, sys
import numpy as np
sys.path.insert(0, %(root)r)
from bench import make_clip
from uhc_b200.agent import BatchedAgent, RolloutBuffer
E, T, out = %(E)d, %(T)d, %(out)r
ex, shape = make_clip()
agent = BatchedAgent(E, [ex], [shape], device=0, seed=1)
agent.reset_envs()
buf = RolloutBuffer(1, E, agent.dev, agent.act_dim, agent.obs_dim)
h = hashlib.sha256()
for t in range(T):
    agent.rollout(buf, 1, 0)
    for x in (agent.obs, buf.actions[0], buf.rewards[0], buf.masks[0], buf.fails[0]):
        h.update(x.cpu().numpy().tobytes())
st = {k: np.ascontiguousarray(np.asarray(v)) for k, v in agent.engine.get_states().items()}
res = dict(envs=E, steps=T, outputs_sha256=h.hexdigest(),
           state_sha256={k: hashlib.sha256(("%%s %%s|" %% (v.dtype.str, v.shape)).encode() + v.tobytes()).hexdigest() for k, v in sorted(st.items())},
           counters=agent.engine.counters)
json.dump(res, open(out, "w"), indent=1, sort_keys=True, default=int)
"""


def digest(so=None, envs=4096, steps=300):
    """The digest of `steps` rollout steps of `envs` envs on the library `so` (None: the production library), as a dict."""
    env = dict(os.environ)
    if so:
        env["UHC_B200_SO"] = so
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "digest.json")
        subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT, E=envs, T=steps, out=out)], env=env, check=True, cwd=ROOT)
        with open(out) as f:
            return json.load(f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON file to write")
    ap.add_argument("--so", default=None, help="library to run (default: the production library)")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=300)
    a = ap.parse_args()
    res = digest(a.so, a.envs, a.steps)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(res, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
