"""CPU: the fp64 reference of the policy half of a rollout step (tests/policy_ref.py) against the reference's own ZFilter and nets (tests/golden),
and the statistics of the counter-based generators.  The GPU tests require the kernels to equal these generators element for element, so the
statistical properties checked here carry over to the GPU's streams."""
import math
import os

import numpy as np
import pytest
import torch
from scipy import stats

from tests import policy_ref as R
from uhc.khrylib.utils.zfilter import RunningStat


@pytest.fixture(scope="module")
def g(golden_dir):
    z = np.load(os.path.join(golden_dir, "ppo_small.npz"))
    return {k: z[k] for k in z.files}


def shape_vector(golden_dir):
    """the 17-dim shape vector (betas + gender) of the goldens' clip: obs columns 640-656, constant while every env holds this subject"""
    z = np.load(os.path.join(golden_dir, "expert_sway.npz"))
    return np.concatenate([z["beta"][0], [z["gender"][0]]]).astype(np.float32)


def test_one_row_batches_equal_running_stat_and_the_golden(g):
    """with one-row batches the batched ZFilter is the reference's per-sample push; it reproduces the z_raw -> z_out trace of khrylib's ZFilter"""
    raw = g["z_raw"]
    st, rs = R.zf_empty(raw.shape[1]), RunningStat(raw.shape[1])
    out = []
    for row in raw:
        st = R.zf_merge(st, row[None])
        rs.push(row)
        assert st[0] == rs.n and np.array_equal(st[1], rs.mean)
        assert np.abs(st[2] - rs._S).max() <= 1e-12 * (1.0 + np.abs(rs._S).max())
        out.append(R.zf_apply(st, row[None])[0])
    # measured: 6.7e-16 (mean), 8.9e-16 (std), 7.7e-14 (normalised rows, |y| <= 5)
    assert st[0] == float(g["z_n"]) and np.abs(st[1] - g["z_mean"]).max() < 1e-13
    assert np.abs(R.zf_std(st) - g["z_std"]).max() < 1e-13
    assert np.abs(np.array(out) - g["z_out"]).max() < 1e-12
    # one batch of all 40 rows has the same moments as 40 pushes (the merge is exact arithmetic up to rounding)
    b = R.zf_merge(R.zf_empty(raw.shape[1]), raw)
    assert np.abs(b[1] - st[1]).max() < 1e-12 and np.abs(R.zf_std(b) - R.zf_std(st)).max() < 1e-12


@pytest.mark.parametrize("M", [1, 2, 3, 17, 200, 1000, 6250])
def test_constant_columns_give_zero_spread_and_zero_output(golden_dir, M):
    sv = shape_vector(golden_dir)
    cols = np.concatenate([sv, np.float32([0.1, -3.7e5, 1e-30, 0.0])])
    x = np.tile(cols, (M, 1))
    st = R.zf_empty(len(cols))
    for _ in range(4):
        st = R.zf_merge(st, x)
        assert np.array_equal(st[1], cols.astype(np.float64)) and (st[2] == 0).all()
        assert (R.zf_apply(st, x) == 0).all()
    assert R.zf_merge(st, x[:0]) is st                       # an empty batch changes nothing


def test_bf16_rounding_is_nearest_even():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(100000).astype(np.float32) * 10.0 ** rng.integers(-6, 6, 100000),
                        # exact ties: the bit below the kept 16 set, nothing under it -> to the even neighbour
                        (np.arange(2000, dtype=np.uint32) << 16 | 0x8000).view(np.float32)[100:],
                        np.float32([0.0, -0.0, 3.0e38, -3.0e38, 1e-40])]).astype(np.float32)
    ref = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(R.bf16_bits(x), ref)


def _golden_nets(g, pre, head):
    keys = [f"net.affine_layers.{i}" for i in range(len(g["hsize"]))] + [head]
    return [g[f"{pre}{k}.weight"] for k in keys], [g[f"{pre}{k}.bias"] for k in keys]


def test_unrounded_mlp_reproduces_the_golden_nets(g):
    mean, _ = R.mlp_forward(*_golden_nets(g, "p0.", "action_mean"), g["states"], "gelu", rounded=False)
    v, _ = R.mlp_forward(*_golden_nets(g, "v0.", "value_head"), g["states"], "gelu", rounded=False)
    # measured: 9e-18 (mean), 1.4e-17 (values)
    assert np.abs(mean - g["mean"]).max() < 1e-14 and np.abs(v - g["values"]).max() < 1e-14


def test_unrounded_mcp_reproduces_the_golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "mcp_ppo.npz"))
    P, hs, nc = int(z["nprim"]), len(z["hsize"]), len(z["composer_dim"]) + 1
    prims = [([z[f"p0.nets.{k}.0.affine_layers.{i}.weight"] for i in range(hs)] + [z[f"p0.nets.{k}.1.weight"]],
              [z[f"p0.nets.{k}.0.affine_layers.{i}.bias"] for i in range(hs)] + [z[f"p0.nets.{k}.1.bias"]]) for k in range(P)]
    comp = ([z[f"p0.composer.0.affine_layers.{i}.weight"] for i in range(nc)], [z[f"p0.composer.0.affine_layers.{i}.bias"] for i in range(nc)])
    mean, w, _ = R.mcp_forward(prims, comp, z["states"], "relu", rounded=False)
    # the golden holds fp32 weights of an fp64 init: measured 1.3e-9 (mean, |mean| <= 0.025), 5.3e-9 (weight)
    assert np.abs(mean - z["mean"]).max() < 1e-8 and np.abs(w - z["weight"]).max() < 3e-8


def test_rounded_forward_stays_near_the_exact_one(g):
    """the rounding points cost about a bf16 ulp of the output scale, no more (a wrong rounding point would be far off or identical)"""
    Ws, bs = _golden_nets(g, "p0.", "action_mean")
    exact, scale = R.mlp_forward(Ws, bs, g["states"], "gelu", rounded=False)
    rnd, _ = R.mlp_forward(Ws, bs, g["states"], "gelu")
    rel = np.abs(rnd - exact).max() / scale.max()
    assert 1e-5 < rel < 2 ** -7, rel


def test_gaussian_logp_matches_the_torch_reference():
    rng = np.random.default_rng(1)
    mean, a, ls = rng.standard_normal((50, 105)), rng.standard_normal((50, 105)), rng.uniform(-3, 1, 105)
    lp, mag = R.gaussian_logp(mean, ls, a)
    ref = torch.distributions.Normal(torch.tensor(mean), torch.tensor(np.exp(ls))).log_prob(torch.tensor(a)).sum(1).numpy()
    assert np.abs(lp - ref).max() < 1e-13 * mag.max()


# ---------------------------------------------------------------------------------------------------------------- generators
N20 = 1 << 20


def test_normals_pass_a_ks_test_and_stop_at_the_tail_cut():
    z, r = R.noise(seed=12345, step=7, M=N20 // 105 + 1, A=105)
    z = z.reshape(-1)[:N20]
    ks = stats.kstest(z, "norm")
    assert ks.pvalue > 1e-3, ks                    # measured p = 0.44
    assert abs(z.mean()) < 5 / math.sqrt(N20) and abs(z.std() - 1.0) < 5 / math.sqrt(N20)
    # u1 >= 2^-24 (1 - 2^-23) cuts the tail at sqrt(2 * 24 ln 2) = 5.7681 sigma (a normal exceeds it with probability 8e-9)
    assert abs(R.TAIL - math.sqrt(2.0 * 24.0 * math.log(2.0))) < 1e-7 and abs(R.TAIL - 5.76811) < 1e-5
    assert np.abs(z).max() <= R.TAIL and r.max() <= R.TAIL
    # u1 runs over (k + 1) fp32(1 / (2^24 + 2)), k = 0 .. 2^24 - 1: never 0 (the log is finite) and never 1
    k = np.array([0, 1, (1 << 23) - 1, (1 << 24) - 2, (1 << 24) - 1], dtype=np.float32)
    u1 = (k + np.float32(1.0)) * R.U1_SCALE
    assert u1[0] == R.U1_SCALE and np.all(np.diff(u1) > 0) and u1[-1] == np.float32(1.0 - 2.0 ** -23) and u1[-1] < 1.0


def _corr(a, b):
    a, b = a.reshape(-1) - a.mean(), b.reshape(-1) - b.mean()
    return float((a * b).sum() / math.sqrt((a * a).sum() * (b * b).sum()))


def test_neighbouring_streams_are_uncorrelated():
    """neighbouring dims, rows, control steps, and the per-rank seeds s, s + 1: each correlation below 5 / sqrt(n)"""
    M, A, seed = 4096, 105, 1000003
    z0, _ = R.noise(seed, 41, M, A)
    z1, _ = R.noise(seed, 42, M, A)
    zs, _ = R.noise(seed + 1, 41, M, A)
    pairs = {"dim": (z0[:, :-1], z0[:, 1:]), "row": (z0[:-1], z0[1:]), "step": (z0, z1), "seed": (z0, zs),
             "row seam": (z0[:-1, -1], z0[1:, 0])}      # the last dim of a row and the first of the next are neighbouring stream indices too
    for name, (a, b) in pairs.items():
        c = _corr(a, b)
        assert abs(c) < 5 / math.sqrt(a.size), (name, c)
    # the same uniforms drive the mean-action flags: neighbouring envs, steps and seeds
    u0, u1, us = R.mean_action_uniform(seed, 41, N20), R.mean_action_uniform(seed, 42, N20), R.mean_action_uniform(seed + 1, 41, N20)
    for name, (a, b) in {"env": (u0[:-1], u0[1:]), "step": (u0, u1), "seed": (u0, us)}.items():
        c = _corr(a.astype(np.float64), b.astype(np.float64))
        assert abs(c) < 5 / math.sqrt(a.size), (name, c)


@pytest.mark.parametrize("noise_rate", [0.3, 0.5])
def test_mean_action_rate(noise_rate):
    f = np.concatenate([R.mean_action_flags(77, s, 4096, noise_rate) for s in range(64)])
    p = 1.0 - noise_rate
    assert abs(f.mean() - p) < 5 * math.sqrt(p * (1 - p) / f.size), f.mean()
    assert R.mean_action_flags(77, 3, 4096, 0.0).all() and not R.mean_action_flags(77, 3, 4096, 1.0).any()


def test_mean_action_threshold_is_formed_in_fp32():
    """1.0f - noise_rate is rounded to fp32 before the compare: a uniform equal to it is NOT a mean-action draw (u < p, not u <= p)"""
    u = R.mean_action_uniform(5, 9, 4096)
    k = int(np.argmax((u > 0.25) & (u < 0.5)))
    nr = float(np.float32(1.0) - u[k])                       # exact: 1 - u[k] is a multiple of 2^-24 in [0.5, 0.75)
    assert np.float32(1.0) - np.float32(nr) == u[k]
    assert R.mean_action_flags(5, 9, 4096, nr)[k] == 0
    assert R.mean_action_flags(5, 9, 4096, nr - 2.0 ** -24)[k] == 1
