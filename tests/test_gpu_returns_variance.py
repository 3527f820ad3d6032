"""GPU: "returns within stochastic variance" (BASELINE north_star).  The same stochastic policy (same weights, same observation normaliser, same noise
scale) rolled out on the product path -- fp32 physics kernel, wgmma bf16 policy forward, device Gaussian sampler, 1024 envs -- and on the reference-pinned
fp64 oracle env with an fp64 numpy policy (48 envs): episode returns, episode lengths and the failure rate must agree within their sampling error."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
KEYS = ("qpos", "qvel", "wbpos", "wbquat", "bquat", "bangvel", "ee_wpos", "com")


def _gelu(x):
    from math import erf
    return 0.5 * x * (1.0 + np.vectorize(erf)(x / np.sqrt(2.0)))


def test_episode_returns_agree_within_sampling_error(golden_dir):
    import torch
    from oracle import oracle as O
    from uhc_b200 import nn
    from uhc_b200.engine import Engine
    z = np.load(os.path.join(golden_dir, "expert_sway.npz"))
    ex = {k: z[k] for k in z.files}
    so = np.concatenate([ex["beta"][0], [ex["gender"][0]]])
    E, n_cpu, T, log_std = 1024, 48, 45, -2.3
    rng = np.random.RandomState(11)
    starts = rng.randint(0, 30, E).astype(np.int32)
    dev = torch.device("cuda", 0)
    eng = Engine(E)
    eng.load_clips([ex], [so])
    obs = eng.reset(start=starts)
    pol = nn.MLPNet(657, (256, 128), 105, "gelu", device=dev, head_name="action_mean", seed=7)
    zf = nn.ZFilter(657, clip=5.0, device=dev)
    zf(obs, update=True)                                    # statistics of the 1024 reset observations, frozen afterwards on both sides
    ls = torch.full((105,), log_std, device=dev)
    ret = torch.zeros(E, device=dev); length = torch.zeros(E, device=dev); alive = torch.ones(E, dtype=torch.bool, device=dev); failed = torch.zeros(E, dtype=torch.bool, device=dev)
    for t in range(T):
        s = zf(obs, update=False)
        a, _ = nn.gaussian_sample(pol.forward_tc(s), ls, 1234, t)
        obs, rew, ci, fail, end, pct = eng.step(a)
        ret += rew * alive; length += alive
        failed |= alive & (fail != 0)
        alive &= (fail == 0) & (end == 0)
    torch.cuda.synchronize()
    g_ret, g_len, g_fail = ret.cpu().numpy(), length.cpu().numpy(), failed.cpu().numpy()
    n, mean, std = zf.n, zf.mean, zf.std
    W = [w.detach().cpu().numpy().astype(np.float64) for w in pol.W]
    B = [b.detach().cpu().numpy().astype(np.float64) for b in pol.b]
    eng.close()

    om = O.Model()
    c_ret, c_len, c_fail = np.zeros(n_cpu), np.zeros(n_cpu), np.zeros(n_cpu, bool)
    nrng = np.random.RandomState(99)
    for i in range(n_cpu):
        env = O.Env(om, {k: ex[k][starts[i]:] for k in KEYS}, so)
        o = env.reset()
        for t in range(T):
            h = np.clip((o - mean) / (std + 1e-8), -5, 5)
            for k in range(len(W)):
                h = W[k] @ h + B[k]
                if k < len(W) - 1:
                    h = _gelu(h)
            act = h + np.exp(log_std) * nrng.standard_normal(105)
            o, r, done, info = env.step(act)
            c_ret[i] += r; c_len[i] += 1
            if done:
                c_fail[i] = info["fail"]
                break

    def zscore(a, b):
        return (a.mean() - b.mean()) / np.sqrt(a.var(ddof=1) / len(a) + b.var(ddof=1) / len(b) + 1e-12)
    msg = dict(gpu_return=(g_ret.mean(), g_ret.std()), cpu_return=(c_ret.mean(), c_ret.std()), gpu_len=g_len.mean(), cpu_len=c_len.mean(),
               gpu_fail=g_fail.mean(), cpu_fail=c_fail.mean())
    assert abs(zscore(g_ret, c_ret)) < 4.0, msg
    assert abs(zscore(g_len, c_len)) < 4.0, msg
    p = (g_fail.sum() + c_fail.sum()) / (E + n_cpu)
    assert abs(g_fail.mean() - c_fail.mean()) < 4.0 * np.sqrt(max(p * (1 - p), 1e-4) * (1 / E + 1 / n_cpu)) + 1e-9, msg
    assert g_ret.mean() > 1.0 and g_len.mean() > 3.0, msg                   # not a degenerate comparison
