"""Every GEMM entry point and helper kernel of mlp_wgmma.cu and nn_kernels.cu, element by element against the fp64 statements of
tests/gemm_ref.py, at the shapes where tiled kernels go wrong (ragged M / N, k-block counts around the 5-stage ring and the split-K threshold, grids
around the SM count, the production dW reduction), on both store paths of the tensor-core epilogue.

  - bounds per element: |got - ref| <= c sum |a||b| for fp32 outputs (c a fraction of (Kp - 1) 2^-24 for the tensor-core products); bf16 outputs between the roundings of ref -/+ tol with few RNE flips; each c
    is in tests/gemm_ref.py with the worst value measured on an H100, and every test prints its worst next to its bound;
  - every output sits at an offset inside a larger allocation filled with 0xFF (NaN in fp32 and bf16); every byte outside its rows x pitch must come
    back unchanged and every promised padding column as zero.  Offsets are multiples of 256 bytes except where a case means to leave the
    16-byte alignment the TMA store needs;
  - paths without atomics give the same bits on two calls;
  - UHC_TC_TMA_STORE is read once per process, so test_per_thread_epilogue_child_process reruns this file with UHC_TC_TMA_STORE=0: every output
    then takes the per-thread stores and the TMA-only entry points must refuse (-2);
  - bf16 outputs that are not 16-byte aligned, and a bf16 pitch below N, are refused (-2) by every entry point with the buffer left untouched.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import gemm_ref as G

pytestmark = pytest.mark.gpu

ACTS = ["none", "gelu", "tanh", "relu", "sigmoid"]
ACT = {"none": 0, "gelu": 1, "tanh": 2, "relu": 3, "sigmoid": 4}
GUARD = 4096                # bytes of poison on either side of every output (a multiple of 256: the offset keeps the output's alignment)
POISON = 0xFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _L():
    from uhc_b200.engine import load_library
    return load_library()


def _err():
    return _L().uhc_last_error().decode()


def _tma():
    return bool(_L().uhc_tc_tma_store_enabled())


def _st():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(None if t is None else t.data_ptr())


class Out:
    """an output [rows][pitch] of `dtype` at GUARD + off bytes inside a poisoned allocation"""

    def __init__(self, rows, pitch, dtype, off=0):
        import torch
        self.esz = torch.empty(0, dtype=dtype).element_size()
        self.n = rows * pitch * self.esz
        self.off = GUARD + off
        self.buf = torch.full((self.off + self.n + GUARD,), POISON, dtype=torch.uint8, device="cuda")
        self.t = self.buf[self.off:self.off + self.n].view(dtype).view(rows, pitch)
        self.ptr = C.c_void_p(self.buf.data_ptr() + self.off)

    def untouched(self):
        return bool((self.buf[:self.off] == POISON).all()) and bool((self.buf[self.off + self.n:] == POISON).all())

    def all_poison(self):
        return bool((self.buf == POISON).all())

    def bits(self):
        import torch
        return self.t.view(torch.int16).cpu().numpy().view(np.uint16)


def _rel(got, ref, scale):
    """max |got - ref| / scale (scale 0: the output must be exact); inf for a non-finite output"""
    import torch
    d = (got.double() - ref).abs()
    if not bool(torch.isfinite(d).all()):
        return float("inf")
    r = torch.where(scale > 0, d / scale.clamp(min=1e-300), torch.where(d > 0, float("inf"), 0.0))
    return float(r.max()) if r.numel() else 0.0


WORST = {}


def _tc(name, got, ref, scale, Kp, ks=1):
    """a tensor-core product's worst error in units of the recursive-summation ceiling, against K_TC / K_SPLIT"""
    _note(f"{name} (of the ceiling)", _rel(got, ref, scale) / G.ceiling(Kp), G.K_SPLIT if ks > 1 else G.K_TC)


def _note(name, value, bound):
    WORST[name] = max(WORST.get(name, 0.0), value)
    assert value <= bound, (name, value, bound)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"worst {k}: {WORST[k]:.3e}")


_CACHE = {}


def _opnd(seed, M, K, Kp=None, mix="mixed", side="a", dtype=None):
    """cached device operand of tests/gemm_ref.py"""
    import torch
    dtype = dtype or torch.bfloat16
    key = (seed, M, K, Kp, mix, side, dtype)
    if key not in _CACHE:
        if M * (Kp or K) > 1 << 26:       # generated in row blocks: the hash's int64 temporaries of a 2048 x 131072 operand would need ~16 GB at once
            blk = (1 << 26) // (Kp or K)
            _CACHE[key] = torch.cat([G.operand(seed, M, K, Kp, mix, side, r0, min(blk, M - r0), "cuda", dtype) for r0 in range(0, M, blk)])
        else:
            _CACHE[key] = G.operand(seed, M, K, Kp, mix, side, device="cuda", dtype=dtype)
    return _CACHE[key]


def _bias(N, seed=7):
    import torch
    return G._normal(seed, torch.zeros(1, dtype=torch.int64, device="cuda"), N, "cuda")[0].contiguous()


def _sync():
    import torch
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------ plain fp32 products


def _fp32_product(M, N, K, off, bias, seed=1):
    import torch
    Kp = G.pad64(K)
    x, W = _opnd(seed, M, K, Kp, side="a"), _opnd(seed + 1, N, K, Kp, side="b")
    b = _bias(N) if bias else None
    z, _, s = G.linear(x, W, b, "none")
    outs = []
    for _ in range(2):
        y = Out(M, N, torch.float32, off)
        rc = _L().uhc_linear_forward_tc(_p(x), _p(W), _p(b), None, y.ptr, M, N, Kp, 0, 0, _st())
        assert rc == 0, _err()
        outs.append(y)
    _sync()
    ks = G.ksplit(M, N, Kp)
    for y in outs:
        assert y.untouched(), (M, N, K, off, "guard band")
        _tc(f"tc fp32{' split-K' if ks > 1 else ''}", y.t, z, s, Kp, ks)
    if ks == 1:                               # split-K partials arrive in any order, through the TMA reduce-add or fp32 atomics
        assert torch.equal(outs[0].t.view(torch.int32), outs[1].t.view(torch.int32)), (M, N, K, off, "not deterministic")
    return ks


@pytest.mark.parametrize("M,N,K,off", G.FP32_CASES)
def test_tc_fp32_product(M, N, K, off):
    _fp32_product(M, N, K, off, bias=(M * N) % 3 == 0)


def test_tc_fp32_production_dw_reduction():
    """dW = dz^T h at the production size, and the 657-wide input layer's dW (split-K) at the same 131072 rows"""
    M, N, R = G.BIG
    _fp32_product(M, N, R, 0, bias=False, seed=11)
    assert _fp32_product(M, 657, R, 0, bias=False, seed=11) > 1


def test_tc_f32_pitched():
    """uhc_linear_forward_tc_f32_pitched: the product at a padded pitch through the TMA engine (split-K included); padding columns zero"""
    import torch
    for M, N, K in G.PITCHED_CASES:
        Kp, ld = G.pad64(K), (N + 3) // 4 * 4
        seed = 11 if K == 131072 else 1
        x, W = _opnd(seed, M, K, Kp, side="a"), _opnd(seed + 1, N if K != 131072 else 1024, K, Kp, side="b")[:N]
        z, s = G.gemm(x, W)
        y = Out(M, ld, torch.float32)
        rc = _L().uhc_linear_forward_tc_f32_pitched(_p(x), _p(W), y.ptr, ld, M, N, Kp, _st())
        if not _tma():
            _sync()
            assert rc == -2 and y.all_poison(), (M, N, K)
            continue
        assert rc == 0, _err()
        _sync()
        assert y.untouched() and bool((y.t[:, N:] == 0).all()), (M, N, K)
        ks = G.ksplit(M, N, Kp)
        _tc(f"tc fp32 pitched{' split-K' if ks > 1 else ''}", y.t[:, :N], z, s, Kp, ks)


# ------------------------------------------------------------------------------------------------------------------ forward with activations
def _bias_near_zero(x, W, N):
    """a bias that puts row 0's pre-activations within fp32 rounding of 0 (the relu / gelu masks decided by the accumulation's last bits); a
    seeded one for a single row, whose outputs would otherwise all be ~0"""
    if x.shape[0] == 1:
        return _bias(N)
    return (-(x[:1].double() @ W.double().T)[0]).float().contiguous()


def _act_ulps(y, z, act):
    """|y - act(z)| of the kernel's own fp32 z in units of 2^-24 max(|z|, 1); relu and none must be exact"""
    import torch
    ya = G.act(act, z.double())
    if not G.Y_ULPS[act]:
        return 0.0 if torch.equal(y.double(), ya) else float("inf")
    return _rel(y, ya, 2.0 ** -24 * torch.clamp(z.double().abs(), min=1.0))


def _check_y(name, act, ybits, yf, z_ref, s, Kp, z_got=None):
    """fp32 y against act of the kernel's own z (or, without z, against act(z_ref) within the accumulation bound); bf16 y bracketed"""
    import torch
    tol = G.LIPSCHITZ * G.bound(Kp) * s + G.Y_ULPS[act] * 2.0 ** -24 * torch.clamp(z_ref.abs(), min=1.0)
    y_ref = G.act(act, z_ref)
    if yf is not None:
        if z_got is not None:
            _note(f"{name} fp32 y {act} (ulps)", _act_ulps(yf, z_got, act), G.Y_ULPS[act])
        else:
            _note(f"{name} fp32 y {act} (of its bound)", _rel(yf, y_ref, tol), 1.0)
    if ybits is not None:
        inside, flips = G.in_bf16_bracket(ybits, y_ref.cpu().numpy(), tol.cpu().numpy())
        assert inside, (name, act, "bf16 y outside its bracket")
        _note(f"{name} bf16 flips", flips, G.BF16_FLIPS)


@pytest.mark.parametrize("act", ACTS)
def test_tc_forward_activations(act):
    """uhc_linear_forward_tc with a bias and an activation: fp32 y (TMA store, or per-thread at N % 4 != 0 / a 4-byte offset) and bf16 y"""
    import torch
    for M, N, K in G.TRAIN_CASES:
        for off in (0, 4):
            Kp, ld = G.pad64(K), G.pad64(N)
            x, W = _opnd(3, M, K, Kp, side="a"), _opnd(4, N, K, Kp, side="b")
            b = _bias_near_zero(x, W, N)
            z_ref, _, s = G.linear(x, W, b, act)
            yf, yb = Out(M, N, torch.float32, off), Out(M, ld, torch.bfloat16)
            assert _L().uhc_linear_forward_tc(_p(x), _p(W), _p(b), yb.ptr, yf.ptr, M, N, Kp, ld, ACT[act], _st()) == 0, _err()
            _sync()
            assert yf.untouched() and yb.untouched() and bool((yb.t[:, N:] == 0).all()), (M, N, K, off)
            _check_y("tc forward", act, yb.bits()[:, :N], yf.t, z_ref, s, Kp)


@pytest.mark.parametrize("act", ACTS)
def test_tc_train_forward(act):
    """uhc_linear_forward_tc_train: z, bf16 y and fp32 y; and _train_t: z, bf16 y and yT with its zero padding columns"""
    import torch
    for M, N, K in G.TRAIN_CASES:
        Kp, ld, Mp = G.pad64(K), G.pad64(N), G.pad64(M)
        x, W = _opnd(5, M, K, Kp, side="a"), _opnd(6, N, K, Kp, side="b")
        b = _bias_near_zero(x, W, N)
        z_ref, _, s = G.linear(x, W, b, act)
        for off in (0, 4):
            z, yf, yb = Out(M, N, torch.float32, off), Out(M, N, torch.float32, off), Out(M, ld, torch.bfloat16)
            assert _L().uhc_linear_forward_tc_train(_p(x), _p(W), _p(b), yb.ptr, yf.ptr, z.ptr, M, N, Kp, ld, ACT[act], _st()) == 0, _err()
            _sync()
            assert z.untouched() and yf.untouched() and yb.untouched() and bool((yb.t[:, N:] == 0).all()), (M, N, K, off)
            _tc("tc train z", z.t, z_ref, s, Kp)
            _check_y("tc train", act, yb.bits()[:, :N], yf.t, z_ref, s, Kp, z.t)
        z, yb, yT = Out(M, N, torch.float32), Out(M, ld, torch.bfloat16), Out(N, Mp, torch.bfloat16)
        rc = _L().uhc_linear_forward_tc_train_t(_p(x), _p(W), _p(b), yb.ptr, yT.ptr, Mp, z.ptr, M, N, Kp, ld, ACT[act], _st())
        _sync()
        if not _tma():
            assert rc == -2 and z.all_poison() and yb.all_poison() and yT.all_poison(), (M, N, K)
            continue
        assert rc == 0, _err()
        assert z.untouched() and yb.untouched() and yT.untouched(), (M, N, K)
        assert bool((yb.t[:, N:] == 0).all()) and bool((yT.t[:, M:] == 0).all()), (M, N, K, "padding")
        assert torch.equal(yT.t[:, :M], yb.t[:, :N].t()), (M, N, K, "yT is not y's transpose")
        _tc("tc train_t z", z.t, z_ref, s, Kp)
        _check_y("tc train_t", act, yb.bits()[:, :N], None, z_ref, s, Kp)
        first = yb.t.clone()
        assert _L().uhc_linear_forward_tc_train_t(_p(x), _p(W), _p(b), yb.ptr, yT.ptr, Mp, z.ptr, M, N, Kp, ld, ACT[act], _st()) == 0, _err()
        _sync()
        assert torch.equal(first.view(torch.int16), yb.t.view(torch.int16)), (M, N, K, "not deterministic")


# ------------------------------------------------------------------------------------------------------------------ fused dX + activation backward
@pytest.mark.parametrize("act", ACTS)
def test_tc_dx_dact(act):
    """uhc_linear_dx_dact_tc: dz_prev = (dz W) act'(z_prev) as bf16 and transposed bf16, db_prev = its column sums"""
    import torch
    for M, K, N in G.DX_CASES:
        Np, Kq, Mp = G.pad64(N), G.pad64(K), G.pad64(M)
        dz, WT = _opnd(8, M, N, Np, side="a"), _opnd(9, K, N, Np, side="b")
        zp = (_opnd(10, M, K, K, mix="normal", dtype=torch.float32) * 1.5).contiguous()
        zp[0, :] = 0.0                                   # act'(0) and the relu mask at 0
        y_ref, sy, db_ref, sdb = G.dx_dact(dz, WT, zp, act)
        h, _ = G.gemm(dz, WT)
        o_dz, o_dzT, o_db = Out(M, Kq, torch.bfloat16), Out(K, Mp, torch.bfloat16), Out(1, K, torch.float32)
        rc = _L().uhc_linear_dx_dact_tc(_p(dz), _p(WT), _p(zp), o_dz.ptr, o_dzT.ptr, o_db.ptr, M, K, Np, Kq, Mp, ACT[act], _st())
        _sync()
        if not _tma():
            assert rc == -2 and o_dz.all_poison() and o_dzT.all_poison() and o_db.all_poison(), (M, K, N)
            continue
        assert rc == 0, _err()
        assert o_dz.untouched() and o_dzT.untouched() and o_db.untouched(), (M, K, N)
        assert bool((o_dz.t[:, K:] == 0).all()) and bool((o_dzT.t[:, M:] == 0).all()), (M, K, N, "padding")
        assert torch.equal(o_dzT.t[:, :M], o_dz.t[:, :K].t()), (M, K, N, "dzT is not dz's transpose")
        tol = G.bound(Np) * sy + G.C_DACT[act] * h.abs() + 2.0 ** -23 * y_ref.abs()
        inside, flips = G.in_bf16_bracket(o_dz.bits()[:, :K], y_ref.cpu().numpy(), tol.cpu().numpy())
        assert inside, (M, K, N, act, "dz outside its bracket")
        _note("dx_dact bf16 flips", flips, G.BF16_FLIPS)
        _note("dx_dact db", _rel(o_db.t[0], db_ref, sdb + h.abs().sum(0)), G.C_DB)


# ------------------------------------------------------------------------------------------------------------------ helper kernels
@pytest.mark.parametrize("act", ACTS)
def test_dact_bf16_both_kernels(act):
    """uhc_dact_bf16: the v4 kernel (N % 4 == 0, aligned) and the scalar one (N % 4 != 0, or a dz 2 bytes off its 8-byte alignment)"""
    import torch
    for M, N, off, z_on in [(129, 128, 0, True), (33, 105, 0, True), (4097, 132, 2, True), (31, 1, 0, True), (64, 64, 0, False), (65, 33, 0, False)]:
        Np, Mp = G.pad64(N), G.pad64(M)
        dh = _opnd(12, M, N, N, mix="mixed", dtype=torch.float32).contiguous()
        z = (_opnd(13, M, N, N, mix="normal", dtype=torch.float32) * 1.5).contiguous() if z_on else None
        if z is not None:
            z[0, :] = 0.0
        y_ref, db_ref, sdb = G.dact_ref(dh, z, act)
        o_dz, o_dzT, o_db = Out(M, Np, torch.bfloat16, off), Out(N, Mp, torch.bfloat16), Out(1, N, torch.float32)
        assert _L().uhc_dact_bf16(_p(dh), _p(z), o_dz.ptr, o_dzT.ptr, o_db.ptr, M, N, Np, Mp, ACT[act], _st()) == 0, _err()
        _sync()
        assert o_dz.untouched() and o_dzT.untouched() and o_db.untouched(), (M, N, off)
        assert bool((o_dz.t[:, N:] == 0).all()) and bool((o_dzT.t[:, M:] == 0).all()), (M, N, off, "padding")
        assert torch.equal(o_dzT.t[:, :M], o_dz.t[:, :N].t()), (M, N, off, "dzT is not dz's transpose")
        tol = (G.C_DACT[act if z_on else "none"] * dh.double().abs() + 2.0 ** -24 * y_ref.abs())
        inside, flips = G.in_bf16_bracket(o_dz.bits()[:, :N], y_ref.cpu().numpy(), tol.cpu().numpy())
        assert inside, (M, N, off, act, "dz outside its bracket")
        _note("dact flips", flips, G.BF16_FLIPS)
        _note("dact db", _rel(o_db.t[0], db_ref, dh.double().abs().sum(0)), G.C_DB)


def test_transpose_bf16_both_kernels_exact():
    """uhc_transpose_bf16: v4 kernel (C, pitches % 4 == 0, 8-byte aligned) and the scalar one; exact, zero padded to ld_out"""
    import torch
    for R_, C_, ld_in, off in [(129, 128, 128, 0), (33, 105, 128, 0), (4097, 657, 704, 0), (64, 64, 64, 2), (1, 1, 8, 0), (127, 32, 32, 0)]:
        a = _opnd(14, R_, C_, ld_in, mix="mixed")
        ld_out = G.pad64(R_)
        o = Out(C_, ld_out, torch.bfloat16, off)
        assert _L().uhc_transpose_bf16(_p(a), o.ptr, R_, C_, ld_in, ld_out, _st()) == 0, _err()
        _sync()
        assert o.untouched(), (R_, C_, off)
        assert torch.equal(o.t[:, :R_].view(torch.int16), G.transpose(a, R_, C_).contiguous().view(torch.int16)), (R_, C_, off)
        assert bool((o.t[:, R_:] == 0).all()), (R_, C_, off, "padding")


# ------------------------------------------------------------------------------------------------------------------ SIMT fp32 GEMM
@pytest.mark.parametrize("act", ACTS)
def test_simt_forward_backward(act):
    """uhc_linear_forward (k_gemm<true, false>, every activation) and uhc_linear_backward (dx: k_gemm<true, true>, dW: k_gemm<false, true>, db)"""
    import torch
    f32 = torch.float32
    for M, N, K in G.SIMT_CASES:
        x, W = _opnd(15, M, K, K, side="a", dtype=f32), _opnd(16, N, K, K, side="b", dtype=f32)
        b = _bias_near_zero(x, W, N)
        z_ref, _, s = G.linear(x, W, b, act)
        y, z = Out(M, N, f32), Out(M, N, f32)
        assert _L().uhc_linear_forward(_p(x), _p(W), _p(b), y.ptr, z.ptr, M, N, K, ACT[act], _st()) == 0, _err()
        _sync()
        assert y.untouched() and z.untouched(), (M, N, K)
        _note("simt z", _rel(z.t, z_ref, s), G.C_SIMT)
        _note(f"simt y {act} (ulps)", _act_ulps(y.t, z.t, act), G.Y_ULPS[act])
        if act != "none":
            continue
        dz = _opnd(17, M, N, N, side="a", dtype=f32)
        dx, dW, db = Out(M, K, f32), Out(N, K, f32), Out(1, N, f32)
        assert _L().uhc_linear_backward(_p(x), _p(W), _p(dz), dx.ptr, dW.ptr, db.ptr, M, N, K, _st()) == 0, _err()
        _sync()
        assert dx.untouched() and dW.untouched() and db.untouched(), (M, N, K)
        r, sr = G.gemm(dz, W.T.contiguous())
        _note("simt dx", _rel(dx.t, r, sr), G.C_SIMT)
        r, sr = G.gemm(dz.T.contiguous(), x.T.contiguous())
        _note("simt dW", _rel(dW.t, r, sr), G.C_SIMT)
        _note("simt db", _rel(db.t[0], dz.double().sum(0), dz.double().abs().sum(0)), G.C_DB)


# ------------------------------------------------------------------------------------------------------------------ refused arguments
def test_refuses_unaligned_bf16_output_and_short_pitch():
    """a bf16 y 2, 4 or 8 bytes off 16-byte alignment, or with ldy < N, is refused (-2) by every entry point that writes one, nothing is written,
    and the library works afterwards"""
    import torch
    M, N, K = 33, 105, 128
    Kp, ld, Mp = G.pad64(K), G.pad64(N), G.pad64(M)
    x, W = _opnd(18, M, K, Kp, side="a"), _opnd(19, N, K, Kp, side="b")
    b = _bias(N)
    L, st = _L(), _st()
    z = Out(M, N, torch.float32)
    yT = Out(N, Mp, torch.bfloat16)
    row0, rows = (C.c_int * 1)(0), (C.c_int * 1)(M)
    Ws, bs = (C.c_void_p * 1)(W.data_ptr()), (C.c_void_p * 1)(b.data_ptr())
    calls = {
        "forward_tc": lambda y, ldy: L.uhc_linear_forward_tc(_p(x), _p(W), _p(b), y, None, M, N, Kp, ldy, ACT["gelu"], st),
        "train": lambda y, ldy: L.uhc_linear_forward_tc_train(_p(x), _p(W), _p(b), y, None, z.ptr, M, N, Kp, ldy, ACT["gelu"], st),
        "train_t": lambda y, ldy: L.uhc_linear_forward_tc_train_t(_p(x), _p(W), _p(b), y, yT.ptr, Mp, z.ptr, M, N, Kp, ldy, ACT["gelu"], st),
        "grouped": lambda y, ldy: L.uhc_linear_forward_tc_grouped(1, row0, rows, _p(x), Ws, bs, y, None, M, N, Kp, ldy, ACT["gelu"], st),
    }
    for name, call in calls.items():
        for off, ldy in [(2, ld), (4, ld), (8, ld), (0, 96)]:
            y = Out(M, ld, torch.bfloat16, off)
            assert call(y.ptr, ldy) == -2, (name, off, ldy)
            assert ("aligned" if off else ">= N") in _err(), (name, off, _err())
            _sync()
            assert y.all_poison() and z.all_poison() and yT.all_poison(), (name, off, ldy)
    y = Out(M, ld, torch.bfloat16)
    assert calls["forward_tc"](y.ptr, ld) == 0, _err()
    _sync()
    z_ref, _, s = G.linear(x, W, b, "gelu")
    _check_y("after refusal", "gelu", y.bits()[:, :N], None, z_ref, s, Kp)


# ------------------------------------------------------------------------------------------------------------------ the other store path
def test_per_thread_epilogue_child_process():
    """this file again in a child process with UHC_TC_TMA_STORE=0 (read once per process): every tensor-core output through the per-thread stores"""
    if os.environ.get("UHC_TC_TMA_STORE") == "0":
        pytest.skip("already the child")
    import torch
    _CACHE.clear()
    torch.cuda.empty_cache()                 # the child needs the device memory this process's operands held
    env = dict(os.environ, UHC_TC_TMA_STORE="0")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider",
                                                                           os.path.abspath(__file__), "-k", "not child_process"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-8000:] + r.stderr[-4000:]
    assert " passed" in r.stdout and " failed" not in r.stdout
