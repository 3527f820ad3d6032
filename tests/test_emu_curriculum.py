"""The device curriculum's rules (uhc_b200/csrc/curriculum_core.h), compiled for the host, against the reference's Python: the freq_dict
update of the training loop (with start frames), failure_weights, and the precision-mode start law against draws of the unmodified
reference (tests/golden/precision_hist.npz, tools/make_golden.py gen_precision)."""
import os

import numpy as np
import pytest
from scipy import stats

from tests.emu import curriculum_emu as E
from uhc_b200.agent import failure_weights

G = os.path.join(os.path.dirname(__file__), "golden", "precision_hist.npz")


def host_update(fd, clip, pct, start, max_freq=50):
    """AgentCopycat._update_freq_dict with the start frame ([percent, fr_start], agent_copycat.py:561,590-603): step-major log order"""
    clip, pct, start = (np.asarray(x).reshape(-1) for x in (clip, pct, start))
    for c, p, s in zip(clip, pct, start):
        if c >= 0:
            fd[int(c)].append((float(p), int(s)))
    return [h[-max_freq:] for h in fd]


def random_log(rs, T, Ed, C, p_end, hot=None):
    clip = np.where(rs.uniform(size=(T, Ed)) < p_end, rs.randint(0, C, (T, Ed)), -1).astype(np.int32)
    if hot is not None:                                     # one clip ends far more than max_freq times in this rollout
        clip[(clip >= 0) & (rs.uniform(size=(T, Ed)) < 0.7)] = hot
    pct = np.where(rs.uniform(size=(T, Ed)) < 0.4, 1.0, rs.uniform(size=(T, Ed))).astype(np.float32)
    return clip, pct, rs.randint(0, 300, (T, Ed)).astype(np.int32)


@pytest.mark.parametrize("M,hot", [(50, None), (50, 3), (7, 0), (1, None)])
def test_ring_update_matches_freq_dict(M, hot):
    rs = np.random.RandomState(M + (hot or 0))
    C = 13
    rings, fd = E.Rings(C, M), [[] for _ in range(C)]
    for it in range(6):
        clip, pct, start = random_log(rs, 16, 64, C, 0.15 if it % 2 or hot is not None else 0.02, hot)
        if hot is not None:
            assert (clip == hot).sum() > M
        rings.append(clip, pct, start)
        fd = host_update([list(h) for h in fd], clip, pct, start, M)
        for c in range(C):
            assert rings.history(c) == fd[c], (it, c)


def ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("C", [10, 333, 3334, 11000])
def test_weights_match_failure_weights(C):
    rs = np.random.RandomState(C)
    hist = [[(1.0 if rs.uniform() < q else float(rs.uniform(0, 0.99)), 0) for _ in range(rs.randint(0, 51))] for q in rs.uniform(size=C)]
    rings = E.Rings(C, 50)
    rings.set(hist)
    for temp, freq in ((0.2, 0.5), (0.05, 0.9), (1.0, 0.0)):
        w, cdf = rings.weights(temp, freq)
        ref = failure_weights([[p for p, _ in h] for h in hist], temp, freq)
        assert ulps(w, ref).max() <= 1, (temp, freq)
        acc, ref_cdf = 0.0, np.zeros(C, np.float32)       # upload_clip_cdf: fp64 running sum of the fp32 weights, stored as fp32
        for i in range(C):
            acc += float(ref[i])
            ref_cdf[i] = acc
        assert ulps(cdf, ref_cdf).max() <= 1


def test_empty_history_keeps_sample_keys_rule():
    lens = np.array([100, 250, 61, 900], np.int32)
    w, cdf = E.Rings(4, 50).weights(0.2, 0.5, t_max=60, clip_len=lens)
    np.testing.assert_array_equal(w, lens // 60 + 1)
    np.testing.assert_array_equal(cdf, np.cumsum(lens // 60 + 1))


def golden_rings(z):
    rings = E.Rings(len(z["lens"]), 50)
    rings.set([[(float(z["pct"][c, j]), int(z["start"][c, j])) for j in range(z["nent"][c])] for c in range(len(z["lens"]))])
    return rings


def chi2_ok(obs, pmf):
    obs = np.asarray(obs, np.float64)
    n = obs.sum()
    assert obs[pmf[:len(obs)] == 0].sum() == 0 if len(obs) <= len(pmf) else True
    m = pmf > 0
    exp = pmf[m] * n
    o = obs[:len(pmf)][m]
    return stats.chisquare(o, exp * o.sum() / exp.sum()).pvalue


def test_precision_start_law_matches_reference_draws():
    z = np.load(G)
    rings, lens, t_min = golden_rings(z), z["lens"], int(z["t_min"])
    for c in range(len(lens)):
        obs = z["seq.start_hist"][c][:lens[c]]
        assert z["seq.start_hist"][c][lens[c]:].sum() == 0
        p = chi2_ok(obs, rings.start_law(c, lens[c], t_min, 0.5))          # sample_seq passes sampling_freq (0.5) to the start draw
        assert p > 1e-4, (c, p)
    for c in z["fit_keys"]:                                                # get_sample_from_key's default sampling_freq 0.75
        p = chi2_ok(z[f"key{c}.start_hist"][:lens[c]], rings.start_law(c, lens[c], t_min, 0.75))
        assert p > 1e-4, (c, p)


def test_precision_law_differs_from_uniform():
    """the golden's failure-weighted starts are far from uniform: the law above is not passing by accident"""
    z = np.load(G)
    rings, lens, t_min = golden_rings(z), z["lens"], int(z["t_min"])
    c = int(z["fit_keys"][0])
    assert chi2_ok(z[f"key{c}.start_hist"][:lens[c]], rings.start_law(c, lens[c], t_min, 0.0)) < 1e-12


def test_clip_histogram_matches_reference_draws():
    z = np.load(G)
    rings = golden_rings(z)
    w, _ = rings.weights(0.2, 0.5)
    obs = z["seq.clip_hist"]
    exp = w.astype(np.float64) / w.astype(np.float64).sum() * obs.sum()
    assert stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue > 1e-4


def test_draw_start_follows_its_law():
    """the sampler's draw from uniforms (the kernel's code path) has the law start_law states"""
    z = np.load(G)
    rings, lens, t_min = golden_rings(z), z["lens"], int(z["t_min"])
    import ctypes as C
    L = E._lib()
    rs = np.random.RandomState(2)
    c = int(z["fit_keys"][1])
    u = rs.uniform(size=(60000, 3)).astype(np.float32)
    draws = [L.emu_cur_draw_start(50, E._i(rings.meta), E._f(rings.pct), E._i(rings.start), c, int(lens[c]), t_min, C.c_float(0.75),
                                  C.c_float(a), C.c_float(b), C.c_float(d)) for a, b, d in u]
    assert chi2_ok(np.bincount(draws, minlength=lens[c]), rings.start_law(c, lens[c], t_min, 0.75)) > 1e-4
