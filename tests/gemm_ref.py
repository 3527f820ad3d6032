"""fp64 statements of the GEMM entry points of mlp_wgmma.cu and nn_kernels.cu, written for the tests, with the per-element accumulation scale their
rounding errors grow with, the operands the tests feed them, and fault injectors that apply to the reference the mistakes a tiled tensor-core GEMM
tends to make.

  - gemm / linear / dx_dact / dact / transpose: what each entry point computes, in float64 on the same bf16-rounded operands the kernel reads, and
    Sigma_k |a_k| |b_k| (+ |b|) per element, computed as the product of the absolute-value matrices;
  - in_bf16_bracket: a bf16 output lies between the RNE roundings of ref - tol and ref + tol (rounding is monotone), and equals RNE(ref) but for a
    bounded fraction of entries;
  - operand: seeded operands from an integer hash, so that any block of rows can be regenerated on any device with the same bits (the CPU tests
    rebuild one tile of the largest GPU case without the rest);
  - faults: drop one 64-wide k-block of a 128 x 128 tile, drop one split-K slice, swap two 8-row groups (a swizzle error), round the output or the
    split partials through bf16, shift one 32-column epilogue chunk by one column.

Everything takes and returns torch tensors and runs on their device.  tests/test_gemm_ref.py checks the statements against direct sums and shows
that every fault exceeds the bounds of tests/test_gpu_gemm_fp64.py by at least 10x; no broken kernel is ever run.
"""
import math

import numpy as np
import torch

from tests import policy_ref as R

BM, BN, BK = 128, 128, 64          # k_linear_tc's output tile and k-block
H100_SMS = 132

# --------------------------------------------------------------------------------------------------------------- bounds
# Each is >= 3x the worst error measured on an H100 80GB HBM3 (SXM, 700 W power limit) by tests/test_gpu_gemm_fp64.py, which prints its worst
# next to it.
# tensor-core products: |got - ref| <= K * ceiling(Kp) * (sum |a||b| + |b|) per element, ceiling(Kp) = (Kp - 1) 2^-24 the recursive-summation bound.
# The wgmma accumulation does not round to nearest: on sums of one sign its error grows linearly with Kp (0.105 of the ceiling, 8.2e-4 of
# sum |a||b|, at Kp = 131072 on all-positive rows), so the bound is a fixed fraction of the ceiling rather than a constant.
K_TC = 0.35                 # one slice (measured 0.106)
K_SPLIT = 0.035             # split-K: each slice reduces Kp / ks, the TMA reduce-add or fp32 atomics add the partials (measured 0.0111)
# SIMT fp32 k_gemm: fp32 operands (products rounded), one fmaf chain per output over K
C_SIMT = 3.5e-6            # dW at R = 4097 (measured 1.0e-6)
# the activation of the kernel's own fp32 pre-activation, in units of 2^-24 max(|z|, 1) (A&S erf for gelu)
Y_ULPS = {"gelu": 10.0, "tanh": 6.0, "sigmoid": 5.0, "relu": 0.0, "none": 0.0}      # (gelu 2.8, tanh 1.6, sigmoid 1.2; relu and none exact)
# the activation derivative on the device against the exact one, |got - ref| / |dh| per element (A&S erf + exp for gelu)
C_DACT = {"gelu": 1e-6, "tanh": 1e-6, "sigmoid": 1e-6, "relu": 0.0, "none": 0.0}  # (a priori: A&S erf to 1.5e-7, a few fp32 ulps)
# fraction of bf16 outputs, among those whose bracket is narrower than half an ulp, that are not RNE(ref) (ref within its bound of a boundary)
BF16_FLIPS = 0.02            # (measured 5.2e-3)
# bias gradients: |db - colsum| / colsum |dz| (fp32 partial sums + atomics)
C_DB = 1e-6                 # (measured 3.1e-7)
LIPSCHITZ = 1.13            # max |act'| over every supported activation (gelu's 1.129)


def ceiling(Kp):
    """the classical recursive-summation bound (Kp - 1) 2^-24: a measured error above it is a finding, not a bound"""
    return (Kp - 1) * 2.0 ** -24


def bound(Kp, ks=1):
    """the per-element bound of a tensor-core product over Kp, relative to sum |a||b| + |b|"""
    return (K_SPLIT if ks > 1 else K_TC) * ceiling(Kp)


# --------------------------------------------------------------------------------------------------------------- host decisions restated
def pad64(n):
    return (n + 63) // 64 * 64


def ksplit(M, N, Kp, sms=H100_SMS):
    """the number of split-K slices linear_tc_impl picks for a plain fp32 product (no bias use restriction: bias is ignored but allowed)"""
    nkb, tiles = Kp // BK, -(-N // BN) * -(-M // BM)
    if nkb < 32:
        return 1
    best, ks = 0.0, 1
    for c in range(1, min(16, nkb // 8) + 1):
        items = tiles * c
        eff = items / (-(-items // sms) * sms)
        if eff > best + 0.02:
            best, ks = eff, c
    return ks


def slices(nkb, ks):
    """k-block ranges [kb0, kb1) of the split-K slices (k_linear_tc's kb0 / nkb)"""
    return [(nkb * z // ks, nkb * (z + 1) // ks) for z in range(ks)]


# --------------------------------------------------------------------------------------------------------------- the GPU tests' shapes
# (M, N, K, off): M / N in {1, 31, 32, 33, 105, 127, 128, 129, 4097}, k-block counts {1, 4, 5, 6, 11, 31, 32, 33}, grids of 131 / 132 / 133 / 265 tiles.
# N % 4 != 0 or off = 4 bytes take the per-thread stores (atomics when split); the rest the TMA store (reduce-add when split).
FP32_CASES = [
    (1, 1, 64, 0), (31, 33, 256, 0), (32, 105, 320, 0), (33, 128, 384, 0), (105, 129, 657, 0), (127, 32, 1984, 0), (128, 31, 2048, 0),
    (129, 128, 2112, 0), (4097, 127, 640, 0), (33, 4097, 128, 0), (128, 32, 2048, 4), (129, 128, 2112, 4), (4097, 128, 704, 4),
    (16763, 128, 4096, 0), (1433, 1408, 4096, 0), (893, 2432, 4096, 0), (893, 2430, 4096, 0), (639, 6780, 2048, 0),
    (2048, 657, 16384, 0), (2048, 660, 16384, 0),
]
BIG = (2048, 1024, 131072)      # the production dW reduction: 2048 x 1024 output, 131072 rows
TRAIN_CASES = [(33, 105, 657), (129, 31, 64), (4097, 129, 320), (128, 2048, 704), (1, 33, 1984)]      # (M, N, K), forward with activations
PITCHED_CASES = [(2048, 657, 16384), (127, 33, 2048), (33, 105, 640), (2048, 657, 131072)]           # (M, N, K) at the pitch N rounded up to 4
DX_CASES = [(33, 128, 105), (129, 32, 2048), (4097, 132, 657), (1, 4, 64), (1433, 1024, 512)]         # (M, K, N) of the fused dX + activation backward
SIMT_CASES = [(33, 105, 657), (129, 1, 64), (4097, 31, 127), (128, 128, 128)]                        # (M, N, K) of the fp32 SIMT GEMM


# --------------------------------------------------------------------------------------------------------------- operands
_M32 = 0xFFFFFFFF


def _mul32(h, c):
    """(h * c) mod 2^32 for 0 <= h < 2^32 without int64 overflow"""
    return (h * (c & 0xFFFF) + (((h * (c >> 16)) & 0xFFFF) << 16)) & _M32


def _mix(h):
    h = h & _M32
    h = h ^ (h >> 16)
    h = _mul32(h, 0x7FEB352D)
    h = h ^ (h >> 15)
    h = _mul32(h, 0x846CA68B)
    return h ^ (h >> 16)


def _normal(seed, rows, K, device):
    """approximately N(0, 1) [len(rows)][K] fp32 (Irwin-Hall of the four bytes of a 32-bit hash of (seed, row, column))"""
    idx = rows.to(torch.int64)[:, None] * K + torch.arange(K, device=device, dtype=torch.int64)[None]
    h = _mix(_mix(idx) ^ ((seed * 0x9E3779B1 + 0x632BE5AB) & _M32))
    s = (h & 255) + ((h >> 8) & 255) + ((h >> 16) & 255) + (h >> 24)
    return ((s - 510).to(torch.float32) / 147.8)


KINDS = ("positive", "normal", "range", "cancel", "normal", "zero", "normal", "positive")   # row r is of kind KINDS[r % 8] in a "mixed" operand


def operand(seed, M, K, Kp=None, mix="normal", side="a", r0=0, rows=None, device="cpu", dtype=torch.bfloat16):
    """[rows][Kp] of `dtype` (rows r0 .. r0 + rows of an M-row operand; zero padded past K): "normal" rows, or every row of the kind KINDS[r % 8]:
    all-positive (|y| = sum |a||b| where two such rows meet), large dynamic range along the row (2^-12 .. 2^12), cancelling (the second half of
    the row is minus the first on side "a", equal to it on side "b": where two such rows meet the exact product is 0), zero."""
    Kp = Kp or pad64(K)
    rows = M - r0 if rows is None else rows
    r = torch.arange(r0, r0 + rows, device=device, dtype=torch.int64)
    v = _normal(seed, r, K, device)
    if mix == "mixed":
        kind = r % 8
        k = torch.arange(K, device=device)
        v = torch.where(((kind == 0) | (kind == 7))[:, None], v.abs(), v)
        rng = torch.exp2(((k * 5 + 3) % 25 - 12).to(torch.float32))
        v = torch.where((kind == 2)[:, None], v * rng[None], v)
        h = K // 2
        if h:
            c = v.clone()
            c[:, h:2 * h] = -c[:, :h] if side == "a" else c[:, :h]
            c[:, 2 * h:] = 0
            v = torch.where((kind == 3)[:, None], c, v)
        v = torch.where((kind == 5)[:, None], torch.zeros_like(v), v)
    out = torch.zeros(rows, Kp, device=device, dtype=dtype)
    out[:, :K] = v.to(dtype)
    return out


# --------------------------------------------------------------------------------------------------------------- references
def act(name, z):
    if name == "gelu":
        return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))
    if name == "tanh":
        return torch.tanh(z)
    if name == "relu":
        return torch.clamp(z, min=0.0)
    if name == "sigmoid":
        return torch.sigmoid(z)
    return z


def dact(name, z):
    """act'(z), exact; relu' = [z > 0]"""
    if name == "gelu":
        return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)
    if name == "tanh":
        return 1.0 - torch.tanh(z) ** 2
    if name == "relu":
        return (z > 0).to(z.dtype)
    if name == "sigmoid":
        s = torch.sigmoid(z)
        return s * (1.0 - s)
    return torch.ones_like(z)


def gemm(a, b):
    """a [M][K] b [N][K] (any dtype) -> (a b^T, |a| |b|^T) in float64"""
    a, b = a.double(), b.double()
    return a @ b.T, a.abs() @ b.abs().T


def linear(x, W, bias, act_name):
    """(z, y, scale) of y = act(x W^T + b), scale = sum_k |x_k||W_jk| + |b_j|"""
    z, s = gemm(x, W)
    if bias is not None:
        z, s = z + bias.double(), s + bias.double().abs()
    return z, act(act_name, z), s


def dx_dact(dz, WT, z_prev, act_name):
    """dz_prev = (dz W) act'(z_prev), its scale (sum |dz||W|) |act'|, and the bias gradient colsum(dz_prev) with its scale colsum of the scale"""
    h, s = gemm(dz, WT)
    d = dact(act_name, z_prev.double())
    y, sy = h * d, s * d.abs()
    return y, sy, y.sum(0), sy.sum(0)


def dact_ref(dh, z, act_name):
    """uhc_dact_bf16: dz = dh act'(z) (z None: dz = dh) and db = colsum(dz), with colsum |dz| as db's scale"""
    dh = dh.double()
    y = dh if z is None else dh * dact(act_name, z.double())
    return y, y.sum(0), y.abs().sum(0)


def transpose(a, R, C):
    """out[c][r] = a[r][c] for the R x C block of a"""
    return a[:R, :C].T


# --------------------------------------------------------------------------------------------------------------- bf16 outputs
def in_bf16_bracket(bits, ref, tol):
    """(inside, flips): whether every bf16 value (uint16 bits) lies between RNE(ref - tol) and RNE(ref + tol), and the fraction of entries whose
    bracket is narrower than half an ulp that are not RNE(ref) (where tol is wider, any value of the bracket is a correct rounding)"""
    ref, tol = np.asarray(ref, np.float64), np.asarray(tol, np.float64)
    v = R.bf16_value(bits).astype(np.float64)
    lo, hi = R.bf16((ref - tol).astype(np.float32)), R.bf16((ref + tol).astype(np.float32))
    ulp = np.exp2(np.floor(np.log2(np.maximum(np.abs(ref), 2.0 ** -126))) - 7)
    det = tol < 0.5 * ulp
    flips = ((bits != R.bf16_bits(ref.astype(np.float32))) & det).sum() / max(det.sum(), 1)
    return bool(((v >= lo) & (v <= hi)).all()), float(flips)


def bf16_ulp(x):
    """the spacing of bf16 values at |x| (2^-133 below the normal range)"""
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126)))
    return torch.exp2(e - 7)


# --------------------------------------------------------------------------------------------------------------- fault injectors (one output tile)
def tile(a, b, ti, tj):
    """the operand rows of output tile (ti, tj) as float64"""
    return a[ti * BM:(ti + 1) * BM].double(), b[tj * BN:(tj + 1) * BN].double()


def fault_drop_kblock(at, bt, kb=0):
    """the tile's product without k-block kb"""
    k = slice(kb * BK, (kb + 1) * BK)
    return at @ bt.T - at[:, k] @ bt[:, k].T


def fault_drop_slice(at, bt, ks, z=0):
    """the tile's product without split-K slice z"""
    k0, k1 = slices(at.shape[1] // BK, ks)[z]
    k = slice(k0 * BK, k1 * BK)
    return at @ bt.T - at[:, k] @ bt[:, k].T


def fault_swap_rows8(y, g0=0, g1=1):
    """8-row groups g0 and g1 of the tile exchanged (rows past the output read as zeros, as a clipped store would leave them)"""
    out = torch.zeros(max(y.shape[0], 8 * (max(g0, g1) + 1)), y.shape[1], dtype=y.dtype, device=y.device)
    out[:y.shape[0]] = y
    a, b = out[8 * g0:8 * g0 + 8].clone(), out[8 * g1:8 * g1 + 8].clone()
    out[8 * g0:8 * g0 + 8], out[8 * g1:8 * g1 + 8] = b, a
    return out[:y.shape[0]]


def fault_round_output(y):
    """the fp32 output rounded through bf16"""
    return y.float().to(torch.bfloat16).double()


def fault_round_partials(at, bt, ks):
    """split-K partial tiles staged in bf16 before they are added"""
    out = torch.zeros(at.shape[0], bt.shape[0], dtype=torch.float64, device=at.device)
    for k0, k1 in slices(at.shape[1] // BK, ks):
        k = slice(k0 * BK, k1 * BK)
        out += (at[:, k] @ bt[:, k].T).float().to(torch.bfloat16).double()
    return out


def fault_shift_chunk(y, c=0):
    """the tile's 32-column epilogue chunk c written one column to the right of where it belongs (its first column left at 0)"""
    out = y.clone()
    lo, hi = 32 * c, min(32 * c + 32, y.shape[1])
    out[:, lo:hi] = 0
    out[:, lo + 1:hi] = y[:, lo:hi - 1]
    return out
