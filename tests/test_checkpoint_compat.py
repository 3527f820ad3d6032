"""CPU: the checkpoint wire format (agent_copycat.py:190-201, :249-260).  `running_state` is a pickled
uhc.khrylib.utils.zfilter.ZFilter; a file written by this repo must load into the REFERENCE's class and a file written by the reference
must load here (checked against a file the reference wrote, tests/golden/zfilter_reference.npz)."""
import os
import pickle

import numpy as np


def test_host_zfilter_matches_running_statistics():
    from uhc.khrylib.utils.zfilter import ZFilter
    rng = np.random.RandomState(0)
    x = rng.normal(1.0, 2.0, (50, 6))
    z = ZFilter((6,), clip=5)
    ys = [z(r) for r in x[:10]]                          # per-sample pushes (the reference's use) ...
    z(x[10:])                                            # ... and one batch merge give the statistics of all 50 rows
    assert z.rs.n == 50 and np.allclose(z.rs.mean, x.mean(0)) and np.allclose(z.rs.var, x.var(0, ddof=1))
    assert np.allclose(ys[0], 0.0)                       # first sample: (x - x) / (|x| + eps)
    z2 = ZFilter.from_stats(50, x.mean(0), ((x - x.mean(0)) ** 2).sum(0), clip=5.0)
    assert np.allclose(z2(x[3], update=False), z(x[3], update=False))
    z3 = pickle.loads(pickle.dumps(z2))
    assert z3.rs._n == 50 and np.allclose(z3.rs._M, z2.rs._M) and np.allclose(z3.rs._S, z2.rs._S) and z3.clip == 5.0


def _pickled_names(blob):
    """every name a pickle carries (module / class names and the attribute names of the object states): what an unpickler of either package resolves"""
    import pickletools
    return sorted({str(arg) for op, arg, _ in pickletools.genops(blob) if op.name in ("GLOBAL", "SHORT_BINUNICODE", "BINUNICODE", "UNICODE")})


def test_running_state_round_trips_through_the_reference_class(golden_dir):
    """The reference's ZFilter pickled after 40 pushes, and the reference class applied to this repo's ZFilter of the same rows (tests/golden/zfilter_reference.npz,
    tools/make_golden.py gen_zfilter_pickle): the reference's file loads here with the same statistics, this repo's file names the same classes and attributes
    (so the reference's unpickler resolves it), and normalises as the reference did."""
    from uhc.khrylib.utils.zfilter import ZFilter
    g = np.load(os.path.join(golden_dir, "zfilter_reference.npz"))
    rng = np.random.RandomState(1)
    x = rng.normal(0.5, 3.0, (40, 657))
    ours = ZFilter.from_stats(40, x.mean(0), ((x - x.mean(0)) ** 2).sum(0), clip=5.0)
    assert np.allclose(g["y_ref"], ours(x[0], update=False))
    blob_ref, blob_ours = g["pickle_ref"].tobytes(), pickle.dumps({"running_state": ours})
    assert _pickled_names(blob_ours) == _pickled_names(blob_ref), (_pickled_names(blob_ours), _pickled_names(blob_ref))
    theirs = pickle.loads(blob_ref)["running_state"]          # unpickles into this repo's stand-in (same module path)
    assert type(theirs).__module__ == "uhc.khrylib.utils.zfilter" and theirs.rs._n == 40
    assert np.allclose(theirs.rs._M, x.mean(0)) and np.allclose(theirs.rs._S, ((x - x.mean(0)) ** 2).sum(0))
