"""CPU: the host-side pieces the multi-rank PPO tests (tests/test_gpu_ppo_multirank.py) rest on.

- The sharded fp64 reference equals the unsharded one: GAE over each rank's [T][E] columns with the advantage normalisation over the union
  is GAE over the [T][W E] rollout normalised as one batch, and the ZFilter increments of the ranks, summed in additive form, merge to the
  Chan merge of every batch.
- split_double / join_double (the fp64 statistics riding an fp32 all-reduce): the digits are integers below 2^18, so the fp32 sum over up to
  32 ranks is exact, and the joined sum is the sum of the ranks' values truncated to 2^-30.
- The gradient tensors' tail holds the 5 (5 + 2 D) floats of the statistics for every observation width the environment configurations give.
"""
import itertools
import types
from fractions import Fraction

import numpy as np
import torch

from tests import policy_ref as P
from tests import ppo_ref as R


def test_sharded_reference_equals_unsharded():
    from uhc_b200 import nn
    g = torch.Generator().manual_seed(1)
    T, E, D = 7, 5, 6
    for W in (2, 3, 4):
        r = torch.rand(T, W * E, generator=g, dtype=torch.float64)
        m = (torch.rand(T, W * E, generator=g) > 0.2).double()
        v = torch.randn(T, W * E, generator=g, dtype=torch.float64)
        last = torch.randn(W * E, generator=g, dtype=torch.float64)
        a_all, r_all = R.gae_te(r, m, v, 0.95, 0.95, last)
        shards = [R.gae_te(r[:, s * E:(s + 1) * E], m[:, s * E:(s + 1) * E], v[:, s * E:(s + 1) * E], 0.95, 0.95, last[s * E:(s + 1) * E]) for s in range(W)]
        assert all(torch.equal(a, a_all[:, s * E:(s + 1) * E]) and torch.equal(rt, r_all[:, s * E:(s + 1) * E]) for s, (a, rt) in enumerate(shards))
        flat = torch.cat([a.reshape(-1) for a, _ in shards])
        mu, sd = flat.mean(), flat.std(unbiased=True)
        ref = R.normalize(a_all)
        for s, (a, _) in enumerate(shards):
            assert torch.allclose((a - mu) / sd, ref[:, s * E:(s + 1) * E], rtol=0, atol=1e-13)
        # ZFilter: every rank merges its own batches; the increments in additive form, summed over the ranks, give the merge of all batches
        batches = [[np.random.RandomState(10 * W + s + 100 * j).normal(3.0, 2.0, (4 + s + j, D)) for j in range(2)] for s in range(W)]
        common = np.random.RandomState(W).normal(-1.0, 1.0, (9, D))
        st0 = P.zf_merge(P.zf_empty(D), common)
        t = lambda st: torch.tensor(np.concatenate([[st[0]], st[1], st[2]]))
        sync = nn.zfilter_to_sums(t(st0), D)
        inc = torch.zeros_like(sync)
        full = st0
        for s in range(W):
            st = st0
            for b in batches[s]:
                st = P.zf_merge(st, b)
                full = P.zf_merge(full, b)
            inc += nn.zfilter_to_sums(t(st), D) - sync
        merged = nn.zfilter_from_sums(sync + inc, D)
        assert merged[0].item() == full[0]
        assert torch.allclose(merged, t(full), rtol=1e-12, atol=1e-12)


def _trunc30(x):
    """x truncated toward zero to a multiple of 2^-30, exactly"""
    f = Fraction(x) * 2 ** 30
    return Fraction(int(f), 2 ** 30)


def test_split_join_double_is_exact_over_up_to_32_ranks():
    from uhc_b200 import nn
    rng = np.random.RandomState(3)
    for W in (1, 2, 3, 7, 32):
        mags = 10.0 ** rng.uniform(-10, 16, (W, 64))
        xs = torch.tensor(mags * rng.choice([-1.0, 1.0], (W, 64)))
        xs[:, 0] = torch.tensor(rng.randint(0, 2 ** 20, W), dtype=torch.float64)      # counts: integers
        xs[:, 1] = 2.0 ** 59 / W - 1.0                                                   # near the top of the range
        planes = [nn.split_double(x) for x in xs]
        assert all(p.dtype == torch.float32 and p.abs().max() < 2 ** 18 and torch.equal(p, p.trunc()) for p in planes)
        s32 = planes[0].clone()
        for p in planes[1:]:
            s32 += p                                                                      # the fp32 all-reduce(sum), in rank order
        assert torch.equal(s32.double(), torch.stack(planes).double().sum(0))          # no rounding in the collective
        joined = nn.join_double(s32)
        for i in range(xs.shape[1]):
            exact = sum(_trunc30(float(x)) for x in xs[:, i])
            got = Fraction(float(joined[i]))
            # the join is one fp64 rounding of the exact sum of the truncated values: within 2^-52 of it, and exact where that sum fits 53 bits
            assert abs(got - exact) <= abs(exact) * Fraction(1, 2 ** 52), (W, i)
            if i == 0:
                assert got == exact == sum(int(x) for x in xs[:, 0])


def test_gradient_tail_fits_the_statistics_of_every_observation_width():
    from uhc_b200 import nn
    from uhc_b200.engine import obs_dim_of
    widths = set()
    for obs_v, no_shape, fut in itertools.product((1, 2, 3, 5, 6), (0, 1), range(0, 11)):
        D = obs_dim_of(types.SimpleNamespace(obs_v=obs_v, no_shape=no_shape, fut_frames=fut))
        widths.add(D)
        assert nn.stats_tail_floats(D) >= 5 * (5 + 2 * D), D
    assert {657, 784, 6400, 6570, 3200, 3285} <= widths
    for D in sorted(widths):
        mlp = nn.MLPNet(D, (8,), 3, device="cpu", seed=0)
        mcp = nn.MCPNet(D, (8,), 3, num_primitive=2, composer_dim=(4,), device="cpu", seed=0)
        for net in (mlp, mcp):
            assert net.gfull.numel() - net.nflat >= 5 * (5 + 2 * D), (D, type(net).__name__)
