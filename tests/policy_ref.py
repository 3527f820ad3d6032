"""A plain fp64 statement of the policy half of a rollout step, written for the tests (numpy, plus ppo_ref's torch activations for the nets).

It restates what the kernels of rollout.cu / nn_kernels.cu / mlp_wgmma.cu compute, not the order they compute it in:
  - the ZFilter with batched semantics (DESIGN.md section 5): exact batch moments (two-pass about the batch's first row), the Chan merge of
    (n, mean, S), then y = clip((x - mean) / (std + 1e-8)) with var = S / (n - 1) for n > 1 and mean^2 otherwise;
  - round-to-nearest-even bf16;
  - the MLP / PolicyMCP forward at the tensor-core path's rounding points: bf16 input row and weights, hidden activations stored as bf16, the last
    layer's output left unrounded; exact-erf GELU, tanh, relu, sigmoid;
  - the counter-based generators: splitmix64, the Box-Muller normal of (seed, stream index) and the Bernoulli draw of k_mean_action, bit for bit
    in uint64, the normal evaluated in fp64;
  - the diagonal Gaussian log-probability.
tests/test_policy_ref.py pins it to the reference's own ZFilter / nets (tests/golden) and checks the generators' statistics; the GPU tests
(tests/test_gpu_policy_parity.py) compare the kernels against it element for element.
"""
import math

import numpy as np
import torch

from tests import ppo_ref

CLIP = 5.0
EPS_STD = 1e-8


# ---------------------------------------------------------------------------------------------------------------- ZFilter
def zf_empty(D):
    return (0.0, np.zeros(D), np.zeros(D))


def batch_moments(x):
    """(n, mean, S) of a batch [M][D], two-pass about the first row: a constant column has mean == that value and S == 0 exactly"""
    x = np.asarray(x, dtype=np.float64)
    d = x - x[0]
    md = d.mean(0)
    return float(len(x)), x[0] + md, ((d - md) ** 2).sum(0)


def zf_merge(state, x):
    """Chan et al. merge of the batch's moments into the running (n, mean, S); an empty batch changes nothing"""
    if len(x) == 0:
        return state
    na, ma, Sa = state
    nb, mb, Sb = batch_moments(x)
    n = na + nb
    dlt = mb - ma
    return (n, ma + dlt * (nb / n), Sa + Sb + dlt * dlt * (na * nb / n))


def zf_std(state):
    n, mean, S = state
    return np.sqrt(S / (n - 1.0)) if n > 1 else np.abs(mean)


def zf_apply(state, x, clip=CLIP):
    """normalised batch in fp64 (before the clip when clip is None)"""
    y = (np.asarray(x, dtype=np.float64) - state[1]) / (zf_std(state) + EPS_STD)
    return y if clip is None else np.clip(y, -clip, clip)


# ---------------------------------------------------------------------------------------------------------------- bf16
def bf16_bits(x):
    """round-to-nearest-even fp32 -> bf16 bit patterns (uint16); NaN -> 0x7FFF"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(np.asarray(x, dtype=np.float32)), np.uint16(0x7FFF), b)


def bf16_value(bits):
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def bf16(x):
    """x rounded to bf16 (nearest even), as fp32"""
    return bf16_value(bf16_bits(x))


# ---------------------------------------------------------------------------------------------------------------- nets
def act(name, z):
    return ppo_ref.act(name, torch.as_tensor(z, dtype=torch.float64)).numpy()


def mlp_forward(Ws, bs, x, htype, head_act="none", rounded=True):
    """the net's output [M][out] in fp64 and the last layer's per-element scale sum_k |W_jk h_k| + |b_j| (what its rounding errors grow with).
    rounded: bf16 input and weights, hidden activations stored as bf16 (the tensor-core path); False = every value exact."""
    r = bf16 if rounded else (lambda v: np.asarray(v, dtype=np.float64))
    h = r(x).astype(np.float64)
    n = len(Ws)
    for i in range(n):
        W, b = r(Ws[i]).astype(np.float64), np.asarray(bs[i], dtype=np.float64)
        if i == n - 1:
            return act(head_act, h @ W.T + b), np.abs(h) @ np.abs(W).T + np.abs(b)
        h = act(htype, h @ W.T + b)
        if rounded:
            h = bf16(h.astype(np.float32)).astype(np.float64)


def softmax(c):
    e = np.exp(c - c.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def mcp_forward(prims, composer, x, htype, rounded=True):
    """PolicyMCP: prims = [(Ws, bs)] per primitive, composer = (Ws, bs) activated after its last layer too.  Returns (mean, weights,
    scale): scale bounds what the primitives' and the composer's last-layer rounding moves the mean by, per element."""
    outs = [mlp_forward(W, b, x, htype, rounded=rounded) for W, b in prims]
    xall = np.stack([o for o, _ in outs])                                      # [P][M][A]
    c, cs = mlp_forward(*composer, x, htype, head_act=htype, rounded=rounded)
    w = softmax(c)
    mean = (w.T[:, :, None] * xall).sum(0)
    spread = np.abs(xall - mean[None]).max(0)                                  # a weight error moves the mean by at most this per unit
    scale = (w.T[:, :, None] * np.stack([s for _, s in outs])).sum(0) + spread * cs.max(1, keepdims=True)
    return mean, w, scale


# ---------------------------------------------------------------------------------------------------------------- generators
U64 = np.uint64
GOLDEN_GAMMA = U64(0x9E3779B97F4A7C15)
U1_SCALE = np.float32(float.fromhex("0x1.fffffcp-25"))   # fp32(1 / (2^24 + 2)) = 2^-24 (1 - 2^-23): u1 = (k + 1) U1_SCALE lies in (0, 1)
TAIL = math.sqrt(-2.0 * math.log(float(U1_SCALE)))      # the largest |normal| the generator can return, ~ sqrt(2 * 24 ln 2)


def splitmix64(x):
    x = np.asarray(x, dtype=U64) + GOLDEN_GAMMA
    x = (x ^ (x >> U64(30))) * U64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> U64(27))) * U64(0x94D049BB133111EB)
    return x ^ (x >> U64(31))


def gauss_uniforms(seed, idx):
    """(u1, u2) of stream index idx, h = splitmix64(seed ^ splitmix64(idx)): u1 = ((h >> 40) + 1) U1_SCALE rounded to fp32, in (0, 1);
    u2 = (h & 0xFFFFFF) 2^-24 in [0, 1).  Both exactly the kernel's fp32 values."""
    h = splitmix64(U64(seed) ^ splitmix64(idx))
    u1 = ((h >> U64(40)).astype(np.float32) + np.float32(1.0)) * U1_SCALE
    return u1.astype(np.float64), (h & U64(0xFFFFFF)).astype(np.float64) * 2.0 ** -24


def gauss(seed, idx):
    """Box-Muller normal (cosine branch) of stream index idx, fp64, and its radius sqrt(-2 ln u1)"""
    u1, u2 = gauss_uniforms(seed, idx)
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * np.pi * u2), r


def sample_index(step, M, A):
    """stream index of (row, dim) at a control step: (step M + row) A + dim, in uint64 (wraps like the kernel's)"""
    rows = np.arange(M, dtype=U64)[:, None]
    dims = np.arange(A, dtype=U64)[None, :]
    with np.errstate(over="ignore"):
        return (U64(step) * U64(M) + rows) * U64(A) + dims


def noise(seed, step, M, A):
    """the [M][A] standard normals k_gauss_sample draws at `step`, and their radii"""
    return gauss(seed, sample_index(step, M, A))


def mean_action_uniform(seed, step, E):
    """k_mean_action's uniform per env: (h >> 40) 2^-24 (exact in fp32), h = splitmix64(seed * gamma ^ splitmix64(step E + e + 0x5bd1e995))"""
    e = np.arange(E, dtype=U64)
    with np.errstate(over="ignore"):
        h = splitmix64((U64(seed) * GOLDEN_GAMMA) ^ splitmix64(U64(step) * U64(E) + e + U64(0x5bd1e995)))
    return ((h >> U64(40)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def mean_action_flags(seed, step, E, noise_rate):
    """the mean-action flags (uint8) of one step: u < 1.0f - noise_rate, the threshold formed in fp32; exps = 1 - flag"""
    p_mean = np.float32(1.0) - np.float32(noise_rate)
    return (mean_action_uniform(seed, step, E) < p_mean).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------- Gaussian head
LOG_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)


def gaussian_logp(mean, log_std, a):
    """sum over the action dims of Normal(mean, exp(log_std)).log_prob(a) [M], and the row's sum of |terms| (its rounding scale)"""
    mean, a = np.asarray(mean, dtype=np.float64), np.asarray(a, dtype=np.float64)
    ls = np.asarray(log_std, dtype=np.float64)
    z = (a - mean) / np.exp(ls)
    terms = [-0.5 * z * z, -ls + 0 * z, np.full_like(z, -LOG_SQRT_2PI)]
    return sum(terms).sum(1), sum(np.abs(t) for t in terms).sum(1)
