"""CPU: the device evaluation's per-frame metrics (uhc_b200/csrc/eval_core.h, host build) against uhc_b200/metrics.py.

metrics.py is pinned to the reference's own smpl_eval.compute_metrics by tests/golden/metrics.npz (tests/test_metrics.py); here the
kernel's code must reproduce metrics.py to 1e-12 relative (1e-12 mm absolute near 0) on that golden, on seeded random episodes and on
adversarial frames."""
import os

import numpy as np
import pytest

from tests.emu import eval_emu
from uhc_b200.metrics import compute_metrics, metrics_from_frames

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")
KEYS = ("root_dist", "mpjpe_g", "mpjpe", "pa_mpjpe", "vel_dist", "accel_dist")


def _check(res, rtol=1e-12, atol=1e-12):
    want = compute_metrics(res)
    got = metrics_from_frames(eval_emu.eval_frames(res["pred"], res["gt"], res["pred_jpos"], res["gt_jpos"]), res["percent"], res["fail_safe"])
    assert set(got) == set(want)
    for k in KEYS:
        assert got[k].shape == want[k].shape, k
        np.testing.assert_allclose(got[k], want[k], rtol=rtol, atol=atol, err_msg=k)
    assert bool(got["succ"][0]) == bool(want["succ"][0])
    return got


def _episode(rng, T, noise=0.05):
    gt_q = rng.normal(0, 1, (T, 76)); gt_q[:, 3:7] /= np.linalg.norm(gt_q[:, 3:7], axis=1, keepdims=True)
    pred_q = gt_q + rng.normal(0, noise, (T, 76))
    gt_j = rng.normal(0, 0.5, (T, 24, 3)) + np.array([0, 0, 1.0])
    pred_j = gt_j + rng.normal(0, noise, (T, 24, 3))
    return dict(pred=pred_q, gt=gt_q, pred_jpos=pred_j.reshape(T, 72), gt_jpos=gt_j.reshape(T, 72), percent=1.0, fail_safe=False)


@pytest.mark.parametrize("case", ["a", "b"])
def test_golden(case):
    z = np.load(GOLDEN)
    res = {k: z[f"{case}.in.{k}"] for k in ("pred", "gt", "pred_jpos", "gt_jpos", "percent", "fail_safe")}
    res["percent"], res["fail_safe"] = float(res["percent"]), bool(res["fail_safe"])
    got = _check(res)
    for k in KEYS:       # and the reference's own outputs, to the bound tests/test_metrics.py holds metrics.py to
        np.testing.assert_allclose(got[k], z[f"{case}.out.{k}"], rtol=1e-9, atol=1e-9, err_msg=k)


@pytest.mark.parametrize("seed", range(6))
def test_random_episodes(seed):
    rng = np.random.RandomState(seed)
    _check(_episode(rng, int(rng.randint(3, 60)), noise=[1e-4, 0.01, 0.3][seed % 3]))


def _rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def _with_joints(rng, gt_j, pred_j):
    T = len(gt_j)
    res = _episode(rng, T)
    res["gt_jpos"], res["pred_jpos"] = gt_j.reshape(T, 72), pred_j.reshape(T, 72)
    return res


def test_pred_equals_gt():
    rng = np.random.RandomState(10)
    res = _episode(rng, 8)
    res["pred"], res["pred_jpos"] = res["gt"].copy(), res["gt_jpos"].copy()
    got = _check(res)
    assert np.abs(got["pa_mpjpe"]).max() < 1e-9 and np.abs(got["root_dist"]).max() < 1e-9


def test_similarity_copy_aligns_to_zero():
    """pred = s R gt + t: PA-MPJPE ~ 0, the other errors are not"""
    rng = np.random.RandomState(11)
    gt_j = rng.normal(0, 0.4, (6, 24, 3))
    pred_j = np.stack([1.7 * g @ _rot(rng).T + rng.normal(0, 2, 3) for g in gt_j])
    got = _check(_with_joints(rng, gt_j, pred_j))
    assert np.abs(got["pa_mpjpe"]).max() < 1e-9 and got["mpjpe"].min() > 1.0


def test_reflected_copy():
    rng = np.random.RandomState(12)
    gt_j = rng.normal(0, 0.4, (6, 24, 3))
    pred_j = gt_j * np.array([-1.0, 1.0, 1.0]) + 0.3
    got = _check(_with_joints(rng, gt_j, pred_j))
    assert got["pa_mpjpe"].min() > 1.0           # a reflection cannot be aligned by a rotation


@pytest.mark.parametrize("noise", [0.0, 1e-3])
def test_collinear_joints(noise):
    """every joint (of both sets) on one line through the root: H has rank 1"""
    rng = np.random.RandomState(13)
    T = 5
    d = rng.normal(size=(T, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    tg = rng.normal(0, 0.3, (T, 24, 1)); tg[:, 0] = 0
    gt_j = tg * d[:, None, :] + rng.normal(0, 1, (T, 1, 3))
    e = d + noise * rng.normal(size=(T, 3)); e /= np.linalg.norm(e, axis=1, keepdims=True)
    pred_j = (1.3 * tg + rng.normal(0, 0.05, (T, 24, 1))) * e[:, None, :] + rng.normal(0, 1, (T, 1, 3))
    _check(_with_joints(rng, gt_j, pred_j))


def test_coplanar_joints():
    rng = np.random.RandomState(14)
    T = 5
    gt_j = rng.normal(0, 0.4, (T, 24, 3)); gt_j[..., 2] = 0.7
    pred_j = gt_j + rng.normal(0, 0.03, (T, 24, 3)); pred_j[..., 2] = 0.5
    _check(_with_joints(rng, gt_j, pred_j))
    pred_j = np.stack([g @ _rot(rng).T for g in gt_j])          # a rotated copy of the plane: PA-MPJPE ~ 0
    got = _check(_with_joints(rng, gt_j, pred_j))
    assert np.abs(got["pa_mpjpe"]).max() < 1e-9


def test_far_translation():
    rng = np.random.RandomState(15)
    res = _episode(rng, 7, noise=0.02)
    off = np.array([1e3, -1e3, 1e3])
    for k in ("pred_jpos", "gt_jpos"):
        res[k] = (res[k].reshape(-1, 24, 3) + off).reshape(-1, 72)
    for k in ("pred", "gt"):
        res[k][:, :3] += off
    _check(res)


def test_root_quaternions_unnormalised_and_negative_w():
    rng = np.random.RandomState(16)
    res = _episode(rng, 9)
    res["pred"][:, 3:7] = rng.normal(0, 3, (9, 4)); res["pred"][:, 3] = -np.abs(res["pred"][:, 3])
    res["gt"][:, 3:7] = rng.normal(0, 0.2, (9, 4)); res["gt"][:, 3] = -np.abs(res["gt"][:, 3])
    res["gt"][0, 3:7] = 1e-9            # |q|^2 below 4 eps: the identity rotation
    _check(res)
