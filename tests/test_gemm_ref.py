"""tests/gemm_ref.py on the CPU: its fp64 statements against direct per-element sums, its operands, its restatement of the host's split-K choice,
and, for every shape and bound tests/test_gpu_gemm_fp64.py uses, that every injected fault exceeds that bound by at least 10x on at least one
element of the faulted tile (the GPU test can see what it is for).  The faults are applied to the reference only."""
import math

import numpy as np
import pytest
import torch
from scipy.special import expit

from tests import gemm_ref as G
from tests import policy_ref as R

DETECT = 10.0


def _direct(a, b):
    """sum_k a_ik b_jk and sum_k |a_ik||b_jk| one element at a time (math.fsum: exactly rounded)"""
    a, b = a.double().numpy(), b.double().numpy()
    y = np.array([[math.fsum(a[i] * b[j]) for j in range(len(b))] for i in range(len(a))])
    s = np.array([[math.fsum(np.abs(a[i] * b[j])) for j in range(len(b))] for i in range(len(a))])
    return y, s


@pytest.mark.parametrize("act", ["none", "gelu", "tanh", "relu", "sigmoid"])
def test_statements_equal_direct_sums(act):
    M, N, K = 9, 7, 70
    x, W = G.operand(1, M, K, mix="mixed", side="a"), G.operand(2, N, K, mix="mixed", side="b")
    b = G._normal(7, torch.zeros(1, dtype=torch.int64), N, "cpu")[0]
    y0, s0 = _direct(x, W)
    z, y, s = G.linear(x, W, b, act)
    assert np.abs(z.numpy() - (y0 + b.double().numpy())).max() <= 1e-13 * (s0.max() + 1)
    assert np.allclose(s.numpy(), s0 + np.abs(b.double().numpy()), rtol=1e-14, atol=0)
    zz = z.numpy()
    exact = {"none": zz, "relu": np.maximum(zz, 0), "tanh": np.tanh(zz), "sigmoid": expit(zz),
             "gelu": np.array([0.5 * v * (1 + math.erf(v / math.sqrt(2))) for v in zz.ravel()]).reshape(zz.shape)}[act]
    assert np.allclose(y.numpy(), exact, rtol=1e-14, atol=1e-300)
    # act' against a central difference of act
    zs = torch.linspace(-4, 4, 161, dtype=torch.float64)
    zs = zs[zs.abs() > 1e-3] if act == "relu" else zs
    fd = (G.act(act, zs + 1e-6) - G.act(act, zs - 1e-6)) / 2e-6
    assert (G.dact(act, zs) - fd).abs().max() < 1e-8
    # dz_prev = (dz W) act'(z_prev), its scale and the bias gradient
    dz, WT = G.operand(3, M, N, mix="mixed", side="a"), G.operand(4, K, N, mix="mixed", side="b")
    zp = G.operand(5, M, K, K, dtype=torch.float32) * 1.5
    h0, sh0 = _direct(dz, WT)
    d = G.dact(act, zp.double()).numpy()
    y, sy, db, sdb = G.dx_dact(dz, WT, zp, act)
    assert np.abs(y.numpy() - h0 * d).max() <= 1e-13 * (sh0.max() + 1)
    assert np.allclose(sy.numpy(), sh0 * np.abs(d), rtol=1e-14, atol=0)
    assert np.abs(db.numpy() - np.array([math.fsum(c) for c in (h0 * d).T])).max() <= 1e-12 * (sdb.max().item() + 1)
    dh = G.operand(6, M, K, K, mix="mixed", dtype=torch.float32)
    r, rdb, rs = G.dact_ref(dh, zp, act)
    assert np.allclose(r.numpy(), dh.double().numpy() * d, rtol=1e-15, atol=0)
    assert np.allclose(rdb.numpy(), r.numpy().sum(0), rtol=1e-12, atol=1e-12) and np.allclose(rs.numpy(), np.abs(r.numpy()).sum(0))
    assert torch.equal(G.transpose(x, 5, 60), x[:5, :60].T)


def test_operands_regenerate_by_row_block_and_have_their_kinds():
    full = G.operand(9, 40, 130, mix="mixed", side="a")
    part = G.operand(9, 40, 130, mix="mixed", side="a", r0=17, rows=11)
    assert full.shape == (40, 192) and (full[:, 130:] == 0).all()
    assert torch.equal(full[17:28].view(torch.int16), part.view(torch.int16))
    b = G.operand(10, 40, 130, mix="mixed", side="b")
    y, s = G.gemm(full, b)
    kind = np.arange(40) % 8
    assert (full[kind == 5] == 0).all()
    assert (full[(kind == 0) | (kind == 7)].float() >= 0).all() and (b[(kind == 0) | (kind == 7)].float() >= 0).all()
    pos = np.ix_((kind == 0) | (kind == 7), (kind == 0) | (kind == 7))
    assert torch.equal(y[pos], s[pos])                  # all-positive rows meet: |y| = sum |a||b|
    assert (y[np.ix_(kind == 3, kind == 3)] == 0).all() and (s[np.ix_(kind == 3, kind == 3)] > 0).all()   # cancelling rows meet: exact 0
    rng = full[kind == 2].float().abs()
    assert (rng.max() / rng[rng > 0].min()) > 2.0 ** 20                                # the dynamic-range rows span > 2^20
    v = G._normal(3, torch.arange(2000), 500, "cpu")
    assert abs(v.mean().item()) < 0.01 and abs(v.std().item() - 1.0) < 0.01
    assert torch.equal(G.bf16_ulp(torch.tensor([1.0, 3.0, -0.5], dtype=torch.float64)), torch.tensor([2.0 ** -7, 2.0 ** -6, 2.0 ** -8], dtype=torch.float64))


def test_split_k_choice_and_bracket_helper():
    assert G.ksplit(2048, 1024, 131072) == 1            # 128 tiles already fill 132 SMs to 97 %
    assert G.ksplit(2048, 657, 131072) == 11            # 96 tiles x 11 slices = 1056 = 8 waves of 132
    assert G.ksplit(129, 128, 2112) == 4 and G.ksplit(127, 32, 1984) == 1
    assert G.slices(33, 4) == [(0, 8), (8, 16), (16, 24), (24, 33)]
    ref = np.array([1.0, 1.0 + 2.0 ** -8, -3.0])
    bits = R.bf16_bits(np.array([1.0, 1.0 + 2.0 ** -7, -3.0], np.float32))
    assert G.in_bf16_bracket(bits, ref, np.full(3, 1e-6)) == (True, 1 / 3)      # a tie: RNE goes to 1.0, the other neighbour lies inside
    assert G.in_bf16_bracket(bits, ref, np.full(3, 0.01)) == (True, 0.0)        # brackets wider than half an ulp: no flip counted
    assert not G.in_bf16_bracket(bits, ref - 0.05, np.full(3, 1e-6))[0]


# ------------------------------------------------------------------------------------------------------------------ faults
def _tile(seed, M, N, K, mix="mixed", dtype=torch.bfloat16, bias=None):
    """tile (0, 0) of the case (its operand rows regenerated alone) with its reference and scale"""
    Kp = G.pad64(K) if dtype == torch.bfloat16 else K
    at = G.operand(seed, M, K, Kp, mix, "a", 0, min(M, G.BM), dtype=dtype).double()
    bt = G.operand(seed + 1, N, K, Kp, mix, "b", 0, min(N, G.BN), dtype=dtype).double()
    y, s = at @ bt.T, at.abs() @ bt.abs().T
    if bias is not None:       # seeded, or "near0": the bias that puts row 0's pre-activations at 0 (test_gpu_gemm_fp64._bias_near_zero)
        if bias == "near0":
            bb = (-(at[:1] @ bt.T)[0]).float().double()
        else:
            bb = G._normal(bias, torch.zeros(1, dtype=torch.int64), N, "cpu")[0][:bt.shape[0]].double()
        y, s = y + bb, s + bb.abs()
    return at, bt, y, s


def _faults(at, bt, y, ks, bias=None):
    f = {"drop k-block": G.fault_drop_kblock(at, bt, 0), "swap 8-row groups": G.fault_swap_rows8(y), "shift chunk": G.fault_shift_chunk(y),
         "round output": G.fault_round_output(y)}
    if bias is not None:
        f["drop k-block"] = f["drop k-block"] + (y - at @ bt.T)                      # the bias is added once, outside the k loop
    if ks > 1:
        f["drop split slice"] = G.fault_drop_slice(at, bt, ks, 0) + (y - at @ bt.T)
        f["round split partials"] = G.fault_round_partials(at, bt, ks) + (y - at @ bt.T)
    return f


def _seen(fault, y, tol):
    """max |fault - y| / tol over the tile (where tol = 0 any change counts as seen)"""
    d = (fault - y).abs()
    return torch.where(tol > 0, d / tol.clamp(min=1e-300), torch.where(d > 0, math.inf, 0.0)).max().item()


# At Kp = 131072 the wgmma accumulation's error reaches 0.1 of the ceiling on sums of one sign, so the per-element bound is wide there: in one slice
# (the production 2048 x 1024 dW) wider than one k-block's contribution (1/2048 of the sum) and than a bf16 rounding of the output; in 11 slices (the
# 657-wide input layer's dW) a dropped k-block and bf16 partials show, but by less than 10x.  These are the faults the check cannot see with the required margin
# at that length; every shorter case sees every fault.  (Asserted below the margin, so that a tighter bound shows up here.)
LOW_MARGIN = {(2048, 1024, 131072): {"drop k-block", "round output"}, (2048, 657, 131072): {"drop k-block", "round split partials"}}


def _check_faults(M, N, K, at, bt, y, c, ks, bias=None):
    for name, f in _faults(at, bt, y, ks, bias).items():
        seen = _seen(f, y, c)
        if name in LOW_MARGIN.get((M, N, K), ()):
            assert seen < DETECT, (M, N, K, name, "now seen by 10x: drop it from LOW_MARGIN")
        else:
            assert seen >= DETECT, (M, N, K, name, seen)


@pytest.mark.parametrize("M,N,K,off", G.FP32_CASES + [G.BIG + (0,), (2048, 657, 131072, 0)])
def test_faults_exceed_the_fp32_product_bounds(M, N, K, off):
    Kp = G.pad64(K)
    ks = G.ksplit(M, N, Kp)
    seed = 11 if K == 131072 else 1
    bias = 7 if (M * N) % 3 == 0 and K != 131072 else None
    at, bt, y, s = _tile(seed, M, N, K, bias=bias)
    assert G.bound(Kp, ks) < G.ceiling(Kp)
    _check_faults(M, N, K, at, bt, y, G.bound(Kp, ks) * s, ks, bias)


@pytest.mark.parametrize("M,N,K", G.PITCHED_CASES)
def test_faults_exceed_the_pitched_product_bounds(M, N, K):
    ks = G.ksplit(M, N, G.pad64(K))
    at, bt, y, s = _tile(11 if K == 131072 else 1, M, N, K)
    _check_faults(M, N, K, at, bt, y, G.bound(G.pad64(K), ks) * s, ks)


@pytest.mark.parametrize("M,N,K", G.TRAIN_CASES)
def test_faults_exceed_the_activation_layer_bounds(M, N, K):
    """the z bound (fp32), and for the bf16 y the bracket: a fault must leave ref -/+ (tol + one bf16 ulp) (shown without an activation)"""
    for seed in (3, 5):
        bias = "near0" if M > 1 else 7
        at, bt, y, s = _tile(seed, M, N, K, bias=bias)
        for name, f in _faults(at, bt, y, 1, bias=bias).items():
            assert _seen(f, y, G.bound(G.pad64(K)) * s) >= DETECT, (M, N, K, name)
            if name != "round output":
                assert _seen(f, y, G.LIPSCHITZ * G.bound(G.pad64(K)) * s + G.bf16_ulp(y)) >= DETECT, (M, N, K, name, "bf16")


@pytest.mark.parametrize("M,K,N", G.DX_CASES)
def test_faults_exceed_the_dx_dact_bounds(M, K, N):
    at, bt, y, s = _tile(8, M, K, N)
    for name, f in _faults(at, bt, y, 1).items():
        if name != "round output":
            assert _seen(f, y, G.bound(G.pad64(N)) * s + G.bf16_ulp(y)) >= DETECT, (M, K, N, name)


@pytest.mark.parametrize("M,N,K", G.SIMT_CASES)
def test_faults_exceed_the_simt_bounds(M, N, K):
    bias = "near0" if M > 1 else 7
    at, bt, y, s = _tile(15, M, N, K, dtype=torch.float32, bias=bias)
    for name, f in _faults(at, bt, y, 1, bias=bias).items():
        assert _seen(f, y, G.C_SIMT * s) >= DETECT, (M, N, K, name)
