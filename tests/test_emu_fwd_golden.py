"""CPU: the smooth phase's forward pass (kin_rne_forward, project_force, collide) of the step kernel's source, compiled as the host emulation in
fp32, gives byte for byte what it gave before the narrow phase and the kinematics were restructured (tests/golden/fwd_pass_fp32.npz, written by
`python -m tests.emu.fwd_emu --write` from the sources before).  The poses include what the bench's rollout may never reach: the 40 contact slots
overflowing, upper-body contacts and exact ties for the deepest hull vertex."""
import numpy as np

from tests.emu import fwd_emu


def test_forward_pass_is_bit_identical_to_the_golden():
    want = np.load(fwd_emu.GOLDEN)
    names, got = fwd_emu.run_cases()
    assert list(want["names"]) == names
    # the fixture covers the narrow phase's edge cases
    assert want["con_overflow"].any() and want["upper_contact"].any() and (want["ncon"] == fwd_emu.MAXCON).any() and (want["ncon"] == 0).any()
    for k, x in got.items():
        w = want[k]
        assert x.dtype == w.dtype and x.shape == w.shape, k
        bad = [n for n, a, b in zip(names, x, w) if a.tobytes() != b.tobytes()]
        assert not bad, "%s differs in %d poses, first %s" % (k, len(bad), bad[:5])
