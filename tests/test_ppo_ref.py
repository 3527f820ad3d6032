"""CPU: the fp64 reference of the PPO update (tests/ppo_ref.py) against traces of the reference's own code (tests/golden, tools/make_golden.py
gen_ppo / gen_mcp).  Every GPU gradient test compares against ppo_ref, so it is pinned here first."""
import os

import numpy as np
import pytest
import torch

from tests import ppo_ref as R


@pytest.fixture(scope="module")
def g(golden_dir):
    z = np.load(os.path.join(golden_dir, "ppo_small.npz"))
    return {k: z[k] for k in z.files}


def _params(g, pre, keys):
    return R.leaves([g[pre + k] for k in keys])


PKEYS = ["net.affine_layers.0.weight", "net.affine_layers.0.bias", "net.affine_layers.1.weight", "net.affine_layers.1.bias",
         "net.affine_layers.2.weight", "net.affine_layers.2.bias", "action_mean.weight", "action_mean.bias"]
VKEYS = PKEYS[:6] + ["value_head.weight", "value_head.bias"]


def test_forward_logp_and_advantages_match_golden(g):
    t = lambda k: torch.as_tensor(g[k], dtype=R.F64)
    pol = _params(g, "p0.", PKEYS)
    val = _params(g, "v0.", VKEYS)
    log_std = t("p0.action_log_std").reshape(-1)
    with torch.no_grad():
        mean = R.mlp(pol, t("states"), "gelu")
        v = R.mlp(val, t("states"), "gelu")
        lp = R.gaussian_logp(mean, log_std, t("actions"))
    # measured: 9e-18 (mean), 1.4e-14 (logp, |logp| ~ 1e2), 0 (advantages, returns)
    assert np.abs(mean.numpy() - g["mean"]).max() < 1e-14
    assert np.abs(v.numpy() - g["values"]).max() < 1e-14
    assert np.abs(lp.numpy() - g["logp"].reshape(-1)).max() < 1e-12
    adv, ret = R.estimate_advantages(t("rewards"), t("masks"), t("values"), float(g["gamma"]), float(g["tau"]))
    assert np.abs(adv.numpy() - g["advantages"].reshape(-1)).max() < 1e-13
    assert np.abs(ret.numpy() - g["returns"].reshape(-1)).max() < 1e-13


def test_three_epoch_update_matches_golden(g):
    """AgentPPO.update_policy, 3 epochs, Adam and the first-step clip: p0 / v0 -> p1 / v1 of the reference's fp64 run"""
    t = lambda k: torch.as_tensor(g[k], dtype=R.F64)
    pol = _params(g, "p0.", PKEYS)
    val = _params(g, "v0.", VKEYS)
    log_std = t("p0.action_log_std").reshape(-1)
    losses, first, _ = R.ppo_update(pol, val, lambda p, x: R.mlp(p, x, "gelu"), lambda p, x: R.mlp(p, x, "gelu"), log_std, t("states"), t("actions"),
                                    t("returns"), t("advantages"), t("exps"), float(g["clip_eps"]), int(g["epochs"]), float(g["policy_lr"]),
                                    float(g["value_lr"]), float(g["grad_clip"]))
    for params, pre0, pre1, keys in ((pol, "p0.", "p1.", PKEYS), (val, "v0.", "v1.", VKEYS)):
        for p, k in zip(params, keys):
            d_ref = g[pre1 + k] - g[pre0 + k]
            d_got = p.detach().numpy() - g[pre0 + k]
            assert np.abs(d_ref).max() > 0, k
            # measured: at most 1.1e-15 against updates of 1.5e-4 (policy) and 9e-4 (value)
            assert np.abs(d_got - d_ref).max() < 1e-13, (k, np.abs(d_got - d_ref).max())
    # epoch 0: every ratio is exactly 1, so the surrogate is -mean(A) over the selected rows
    sel = g["exps"] != 0
    assert abs(losses[0][0] + g["advantages"].reshape(-1)[sel].mean()) < 1e-12
    assert all(np.isfinite(l).all() for l in losses)


def test_golden_first_policy_gradient_is_below_the_clip_norm(g):
    """the fixture's first policy gradient has norm 5.53, below the clip norm 40: the golden update never exercises the clip, so the GPU tests
    (tests/test_gpu_grad_parity.py) build their own cases with the clip active"""
    t = lambda k: torch.as_tensor(g[k], dtype=R.F64)
    pol = _params(g, "p0.", PKEYS)
    val = _params(g, "v0.", VKEYS)
    _, (gp, _), _ = R.ppo_update(pol, val, lambda p, x: R.mlp(p, x, "gelu"), lambda p, x: R.mlp(p, x, "gelu"),
                                 t("p0.action_log_std").reshape(-1), t("states"), t("actions"), t("returns"), t("advantages"), t("exps"),
                                 float(g["clip_eps"]), 1, float(g["policy_lr"]), float(g["value_lr"]), float(g["grad_clip"]))
    norm = float(torch.sqrt(sum((x ** 2).sum() for x in gp)))
    assert abs(norm - 5.532) < 1e-3, norm
    assert R.clip_scale(gp, 40.0) == 1.0 and abs(R.clip_scale(gp, 2.0) - 2.0 / (norm + 1e-6)) < 1e-15


def test_mcp_forward_matches_golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "mcp_ppo.npz"))
    P, hs = int(z["nprim"]), len(z["hsize"])
    prims = [R.leaves([z[f"p0.nets.{k}.0.affine_layers.{i}.{w}"] for i in range(hs) for w in ("weight", "bias")] +
                      [z[f"p0.nets.{k}.1.weight"], z[f"p0.nets.{k}.1.bias"]]) for k in range(P)]
    comp = R.leaves([z[f"p0.composer.0.affine_layers.{i}.{w}"] for i in range(len(z["composer_dim"]) + 1) for w in ("weight", "bias")])
    with torch.no_grad():
        mean, w = R.mcp(prims, comp, torch.as_tensor(z["states"], dtype=R.F64), "relu")
        lp = R.gaussian_logp(mean, torch.full((z["actions"].shape[1],), -2.3, dtype=R.F64), torch.as_tensor(z["actions"]))
    # the golden keeps the weights in fp32 (the fp64 init rounded): measured 1.3e-9 (mean, |mean| <= 0.025), 5.3e-9 (weight), 7.4e-8 (logp, |logp| ~ 80)
    assert np.abs(mean.numpy() - z["mean"]).max() < 1e-8
    assert np.abs(w.numpy() - z["weight"]).max() < 3e-8
    assert np.allclose(w.sum(1).numpy(), 1.0, atol=1e-14)
    assert np.abs(lp.numpy() - z["logp"].reshape(-1)).max() < 5e-7


def test_lock_step_gae_equals_per_column_scan():
    """the [T][E] form: each env column is one trajectory of estimate_advantages with V(s_T) added to the last row's delta"""
    gen = torch.Generator().manual_seed(0)
    T, E, gamma, tau = 9, 5, 0.95, 0.9
    r, v = torch.rand(T, E, generator=gen, dtype=R.F64), torch.randn(T, E, generator=gen, dtype=R.F64)
    m = (torch.rand(T, E, generator=gen) > 0.3).to(R.F64)
    last = torch.randn(E, generator=gen, dtype=R.F64)
    adv, ret = R.gae_te(r, m, v, gamma, tau, last)
    for e in range(E):
        r2 = r[:, e].clone()
        r2[-1] += gamma * last[e] * m[-1, e]
        a1, _ = R.gae_te(r2[:, None], m[:, e:e + 1], v[:, e:e + 1], gamma, tau)
        assert torch.allclose(adv[:, e], a1[:, 0], atol=1e-14, rtol=0)
    assert torch.equal(ret, v + adv)
