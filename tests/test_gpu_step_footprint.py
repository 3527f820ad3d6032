"""GPU: k_env_step's per-substep code was made smaller (loops rolled) without changing one floating-point operation or its order.
300 rollout steps of the bench's 4096 envs must give the digest tests/golden/step_digest.json holds: every step's observations, actions,
rewards, masks and fail flags, and the env state records at the end.  The digest was written by scripts/step_digest.py from the library
before the change."""
import json
import os
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def _golden():
    import step_digest
    with open(step_digest.GOLDEN) as f:
        return json.load(f)


def _check(got, want):
    assert (got["envs"], got["steps"]) == (want["envs"], want["steps"])
    assert got["outputs_sha256"] == want["outputs_sha256"], "a step's outputs differ from the digest"
    for k, v in want["state_sha256"].items():
        assert got["state_sha256"][k] == v, k
    assert got["counters"] == want["counters"]


def test_production_library_steps_to_the_digest():
    import step_digest
    from uhc_b200 import build
    want = _golden()
    _check(step_digest.digest(build.build(), want["envs"], want["steps"]), want)
