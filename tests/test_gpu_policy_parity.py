"""GPU: the policy half of a rollout step against its fp64 statement (tests/policy_ref.py), element for element.

Covered: the ZFilter update and apply (uhc_zfilter, uhc_zfilter_ws), the bf16 copy the first GEMM reads, the Gaussian sampler's stream of normals,
the mean-action draws of k_mean_action, the policy forward as uhc_policy_forward(_mcp) and uhc_rollout run it, and the tensor-core GEMM epilogue one layer
at a time.  Bounds are each >= 3x the worst error measured on an H100 80GB HBM3, the measurement beside it; results that are exact by construction
(the bf16 copy, constant columns, the mean-action flags and rows) are compared for equality.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests import policy_ref as R

pytestmark = pytest.mark.gpu

OBS, ACT = 657, 105
SHAPE_COLS = slice(640, 657)         # betas + gender in obs v2: constant while every env holds one subject
SEED = 1000003 * 3 + 1
STEP0 = (1 << 33) + 12345            # (step M + row) A + dim passes 2^32 at every step used here


def _lib():
    from uhc_b200 import nn
    L = nn._lib()
    L.uhc_rollout_last_error.restype = C.c_char_p
    return L


def _st():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else None)


def _cuda(a, dtype=None):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda", dtype=dtype)


def _shape_vector():
    from tests.conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "expert_sway.npz"))
    return np.concatenate([z["beta"][0], [z["gender"][0]]]).astype(np.float32)


SHAPE = _shape_vector()


@pytest.fixture(scope="module")
def shape_vec():
    return SHAPE


@pytest.fixture(scope="module")
def clip(golden_dir):
    z = np.load(os.path.join(golden_dir, "expert_sway.npz"))
    ex = {k: z[k] for k in z.files}
    return ex, np.concatenate([ex["beta"][0], [ex["gender"][0]]])


# ---------------------------------------------------------------------------------------------------------------- ZFilter
KINDS = ("const", "zero", "offset", "heavy", "clipped", "normal")


def column_kinds(D):
    kinds = np.array([KINDS[j % len(KINDS)] for j in range(D)], dtype=object)
    if D >= 657:
        kinds[SHAPE_COLS] = "const"
    return kinds


def make_batch(rng, M, kinds, upd):
    """fp32 batch [M][D]: constant non-zero columns (the shape vector's values; columns 640-656 are the vector itself), exact zeros, a +1e3 offset with
    1e-3 spread, heavy tails (Student t, 2 dof), columns far outside the loaded statistics (mostly clipped at +-5) and plain normals"""
    x = rng.standard_normal((M, len(kinds)), dtype=np.float32)
    c = kinds == "const"
    x[:, c] = const_values(kinds)[c]
    x[:, kinds == "zero"] = 0.0
    o = kinds == "offset"
    x[:, o] = 1e3 + 1e-3 * x[:, o]
    h = kinds == "heavy"
    x[:, h] = rng.standard_t(2, (M, int(h.sum()))).astype(np.float32) * 3.0
    k = kinds == "clipped"
    x[:, k] = 40.0 + 8.0 * x[:, k] + upd
    return x


def const_values(kinds):
    """the value of each constant column: the shape vector itself at 640-656, its entries cycled elsewhere"""
    j = np.arange(len(kinds))
    return np.where((j >= 640) & (j < 657), SHAPE[(j - 640) % 17], SHAPE[j % 17]).astype(np.float32)


def loaded_stats(kinds):
    """statistics as load_sums would restore them from a checkpoint: n = 1e6, and for the 'clipped' columns mean 0, std 1 (the batches sit near 40)"""
    D = len(kinds)
    mean = np.linspace(-0.5, 0.5, D)
    S = np.full(D, 1e6 - 1.0) * np.linspace(0.5, 2.0, D)
    cv = const_values(kinds)
    for j, k in enumerate(kinds):
        if k == "const":                     # a constant column keeps S == 0 only when the loaded history saw the same value
            mean[j], S[j] = cv[j], 0.0
        elif k == "zero":
            mean[j], S[j] = 0.0, 0.0
        elif k == "offset":
            mean[j], S[j] = 1e3, 1e-6 * (1e6 - 1.0)
        elif k == "clipped":
            mean[j], S[j] = 0.0, 1e6 - 1.0
    return (1e6, mean, S)


def ulp32(v):
    return np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


# bounds (worst measured on an H100 80GB HBM3 in parentheses; repeated runs gave identical errors)
ZF_MEAN_REL = 1e-14      # |d mean| / (|mean| + std)  (2.0e-15)
# |d S| / (S + sum of x^2 over the batches merged): the kernel forms a batch's spread as sum x^2 - n mean^2 from raw fp64 sums, so its rounding
# scales with the raw second moment, not with S (a column with a +1e3 offset and 1e-3 spread carries 1e12 times more)  (1.1e-14)
ZF_S_REL = 4e-14
ZF_Y_ULP = 1.0           # fp32 ulps of the fp64 normalisation with the device's statistics  (0.5: correctly rounded)


def check_zfilter(st_gpu, y_gpu, ref, x, kinds, tag, raw2):
    """asserts the device statistics against the fp64 state `ref` after the same batches (raw2: sum of x^2 over those batches, per column) and
    the device's normalised batch against the fp64 normalisation with the device's statistics; returns the worst (mean, S, y) errors"""
    D = len(kinds)
    n, mean, S = ref
    s = st_gpu.cpu().numpy()
    g_mean, g_S = s[1:1 + D], s[1 + D:]
    assert s[0] == n, (tag, s[0], n)
    assert (g_S >= 0).all() and np.isfinite(s).all(), (tag, np.flatnonzero(~(g_S >= 0))[:20])
    const = (kinds == "const") | (kinds == "zero")
    assert (g_S[const] == 0).all(), (tag, "S of constant columns", np.flatnonzero(const & (g_S != 0)))
    std = R.zf_std(ref)
    e_mean = (np.abs(g_mean - mean) / (np.abs(mean) + std + 1e-300)).max()
    e_S = (np.abs(g_S - S) / (S + raw2 + 1e-300)).max()
    assert e_mean <= ZF_MEAN_REL and e_S <= ZF_S_REL, (tag, e_mean, e_S)
    if y_gpu is None:
        return e_mean, e_S, 0.0
    y = y_gpu.cpu().numpy().astype(np.float64)
    yr = R.zf_apply((s[0], g_mean, g_S), x, clip=None)
    assert np.isfinite(y).all(), tag
    bad = const[None, :] & (y != 0)
    assert not bad.any(), (tag, "constant columns normalise to", sorted(set(np.flatnonzero(bad.any(0)))), y[bad][:8])
    cl = np.abs(yr) > R.CLIP * (1 + 1e-6)
    assert (y[cl] == np.sign(yr[cl]) * R.CLIP).all(), (tag, "clipped entries")
    inside = ~cl
    yri = np.clip(yr, -R.CLIP, R.CLIP)
    e_y = (np.abs(y - yri)[inside] / ulp32(yri[inside])).max() if inside.any() else 0.0
    assert e_y <= ZF_Y_ULP, (tag, "y ulps", e_y)
    return e_mean, e_S, e_y


def zf_call(L, x, y, M, D, stats, ws=None):
    if ws is None:
        return L.uhc_zfilter(_p(x), _p(y), M, D, _p(stats), C.c_float(R.CLIP), 1, _st())
    return L.uhc_zfilter_ws(_p(x), _p(y), M, D, _p(stats), C.c_float(R.CLIP), 1, _p(ws), _st())


ZF_M = (1, 2, 15, 16, 17, 200, 1000, 4095, 4096, 4097, 6250, 65536)


@pytest.mark.parametrize("D", [1, 31, 33, 401, 657, 784])
def test_zfilter_against_fp64_merge(D, shape_vec):
    """consecutive updates of uhc_zfilter and uhc_zfilter_ws (bit-identical to each other) from empty and from loaded statistics"""
    import torch
    L = _lib()
    kinds = column_kinds(D)
    rng = np.random.default_rng(D)
    ws = torch.empty(L.uhc_zfilter_workspace_doubles(D), device="cuda", dtype=torch.float64)
    worst = np.zeros(3)
    for start in ("empty", "loaded"):
        for M in ZF_M:
            if M == 65536 and (D != 657 or start == "loaded"):
                continue
            ref = R.zf_empty(D) if start == "empty" else loaded_stats(kinds)
            st = torch.zeros(1 + 2 * D, device="cuda", dtype=torch.float64)
            if start == "loaded":
                from uhc_b200.nn import ZFilter
                zf = ZFilter(D, clip=R.CLIP)
                zf.load_sums(*ref)
                st.copy_(zf.stats)
            st2 = st.clone()
            raw2 = np.zeros(D)
            for upd in range(2 if M == 65536 else 3):
                x = make_batch(rng, M, kinds, upd)
                xd = _cuda(x)
                y, y2 = torch.empty_like(xd), torch.empty_like(xd)
                assert zf_call(L, xd, y, M, D, st) == 0 and zf_call(L, xd, y2, M, D, st2, ws) == 0
                torch.cuda.synchronize()
                assert torch.equal(st, st2) and torch.equal(y, y2), (D, M, start, upd)
                ref = R.zf_merge(ref, x)
                raw2 += (x.astype(np.float64) ** 2).sum(0)
                worst = np.maximum(worst, check_zfilter(st, y, ref, x, kinds, (D, M, start, upd), raw2))
        # an empty batch leaves the statistics alone (and writes nothing)
        before = st.clone()
        for call in (lambda: zf_call(L, xd, None, 0, D, st), lambda: zf_call(L, xd, None, 0, D, st, ws)):
            assert call() in (0, -2)
            torch.cuda.synchronize()
            assert torch.equal(st, before) and torch.isfinite(st).all()
    print(f"zfilter D={D}: worst mean rel {worst[0]:.2e}, S rel {worst[1]:.2e}, y ulps {worst[2]:.2f}")


@pytest.mark.parametrize("M", [200, 1000, 3000, 6250])
def test_shape_vector_columns_normalise_to_zero(M, shape_vec):
    """obs columns 640-656 (the goldens' shape vector, constant over every env) over 20 updates: S stays 0 and the columns normalise to 0, as the
    reference's RunningStat gives -- not to -5 (a negative rounding residue in S made sqrt(S) NaN, and the clip turned NaN into -5)"""
    import torch
    from uhc_b200.nn import ZFilter
    rng = np.random.default_rng(M)
    zf = ZFilter(OBS, clip=R.CLIP)
    failing = set()
    for _ in range(20):
        x = rng.standard_normal((M, OBS), dtype=np.float32)
        x[:, SHAPE_COLS] = shape_vec
        y = zf(_cuda(x)).cpu().numpy()
        S = zf.stats[1 + OBS:].cpu().numpy()
        failing |= set((np.flatnonzero((y[:, SHAPE_COLS] != 0).any(0) | (S[SHAPE_COLS] != 0)) + 640).tolist())
    torch.cuda.synchronize()
    assert not failing, f"E = {M}: columns {', '.join(map(str, sorted(failing)))} do not normalise to 0"
    assert np.array_equal(zf.mean[SHAPE_COLS], shape_vec.astype(np.float64)) and np.isfinite(zf.std).all()


# ---------------------------------------------------------------------------------------------------------------- sampler
SAMPLE_ULPS = 9.0        # |eps - eps_ref| in fp32 ulps (2^-24) of the radius sqrt(-2 ln u1)  (2.8)
LOGP_REL = 5e-7          # of the row's sum of |terms|  (1.5e-7)


@pytest.mark.parametrize("A", [105, 315])
def test_gaussian_sample_is_the_fp64_box_muller_stream(A):
    """uhc_gaussian_sample with mean 0 and log_std 0 returns the noise itself: per element against the fp64 generator, at steps up to 2^40 (stream
    indices past 2^32); logp against the fp64 log-prob of the returned action; mean-action rows equal the mean bit for bit"""
    import torch
    from uhc_b200 import nn
    worst_eps, worst_lp = 0.0, 0.0
    for M in (1, 31, 4097):
        for step in (0, 3, (1 << 32) // (M * A) + 1, 1 << 40):
            mean = torch.zeros(M, A, device="cuda")
            ls = torch.zeros(A, device="cuda")
            a, lp = nn.gaussian_sample(mean, ls, SEED, step)
            eps, r = R.noise(SEED, step, M, A)
            err = np.abs(a.cpu().numpy().astype(np.float64) - eps) / (np.maximum(r, 2.0 ** -12) * 2.0 ** -24)
            worst_eps = max(worst_eps, err.max())
            lref, mag = R.gaussian_logp(np.zeros((M, A)), np.zeros(A), a.cpu().numpy())
            worst_lp = max(worst_lp, (np.abs(lp.cpu().numpy() - lref) / mag).max())
    assert worst_eps <= SAMPLE_ULPS and worst_lp <= LOGP_REL, (worst_eps, worst_lp)
    # a real mean / log_std: the action is mean + exp(log_std) eps; mean-action rows are the mean, logp = -sum log_std - A ln sqrt(2 pi)
    rng = np.random.default_rng(A)
    M = 4097
    mean = _cuda(rng.standard_normal((M, A)).astype(np.float32))
    ls = _cuda(rng.uniform(-2.5, -0.5, A).astype(np.float32))
    flags = rng.integers(0, 2, M).astype(np.uint8)
    a, lp = nn.gaussian_sample(mean, ls, SEED, STEP0, mean_action=_cuda(flags))
    a, lp, mu, lsn = a.cpu().numpy(), lp.cpu().numpy(), mean.cpu().numpy(), ls.cpu().numpy()
    det = flags == 1
    assert np.array_equal(a[det], mu[det])
    eps, _ = R.noise(SEED, STEP0, M, A)
    want = mu.astype(np.float64) + np.exp(lsn.astype(np.float64)) * eps
    e_a = (np.abs(a - want) / (ulp32(want) + np.exp(lsn) * 2.0 ** -24 * SAMPLE_ULPS * R.TAIL))[~det].max()
    assert e_a <= 1.0, e_a
    lref, mag = R.gaussian_logp(mu, lsn, a)
    e_lp = (np.abs(lp - lref) / mag).max()
    assert e_lp <= LOGP_REL and np.abs(lref[det] - (-lsn.astype(np.float64).sum() - A * R.LOG_SQRT_2PI)).max() < 1e-12
    print(f"sampler A={A}: worst eps {worst_eps:.2f} ulps of the radius, logp {max(worst_lp, e_lp):.2e} of sum|terms|, action {e_a:.2f} of its bound")


# ---------------------------------------------------------------------------------------------------------------- policy half through the C ABI
# |mean - mean_ref| / (sum |W| |h| of the last layer), per element  (6.3e-4).  Not round-off of the last layer alone: a hidden activation whose fp32
# value sits near a bf16 rounding boundary lands on the other side in the kernel now and then (3e-4 of the first layer's), and each such
# flip moves the next layer's inputs, so the flips compound to ~6 % of the third layer's activations.
MEAN_REL = 2e-3


def _engine(E, clip, **cfg):
    from uhc_b200.engine import Engine
    eng = Engine(E, **cfg)
    ex, so = clip
    eng.load_clips([ex], [so])
    return eng


def _mlp_weights(net):
    return [w.cpu().numpy() for w in net.W], [b.cpu().numpy() for b in net.b]


def _obs(rng, E, shape_vec):
    x = (rng.standard_normal((E, OBS)) * rng.uniform(0.1, 3.0, OBS) + rng.uniform(-1, 1, OBS)).astype(np.float32)
    x[:, SHAPE_COLS] = shape_vec
    x[:, 5] = 1e3 + 1e-3 * x[:, 5]
    return x


def _forward(L, eng, pol_struct, mcp, obs, ls, stats, update, flags, step=None):
    import torch
    E = obs.shape[0]
    state = torch.full((E, OBS), float("nan"), device="cuda")
    act = torch.full((E, ACT), float("nan"), device="cuda")
    lp = torch.full((E,), float("nan"), device="cuda")
    if step is not None:
        assert L.uhc_rollout_set_step(eng.h, C.c_ulonglong(step)) == 0
    fn = L.uhc_policy_forward_mcp if mcp else L.uhc_policy_forward
    rc = fn(eng.h, _p(obs), C.byref(pol_struct), _p(ls), _p(stats), C.c_float(R.CLIP), C.c_int(update), C.c_ulonglong(SEED), _p(flags), _p(state), _p(act), _p(lp), _st())
    assert rc == 0, L.uhc_rollout_last_error()
    torch.cuda.synchronize()
    return state, act, lp


def check_policy_call(L, eng, pol_struct, mcp, ref_fn, obs_np, shape_vec, rng, tag):
    """one uhc_policy_forward(_mcp) call with a ZFilter update from loaded statistics, then a mean-action call and a sampled call with the
    statistics frozen: state_out, the mean, the sampled action and logp against the fp64 statement"""
    import torch
    from uhc_b200.nn import ZFilter
    E = obs_np.shape[0]
    kinds = np.array(["normal"] * OBS, dtype=object)
    kinds[SHAPE_COLS] = "const"
    zref = (5e3, np.concatenate([np.zeros(640), shape_vec, []]).astype(np.float64), np.concatenate([np.full(640, 2e3), np.zeros(17)]))
    zf = ZFilter(OBS)
    zf.load_sums(*zref)
    obs = _cuda(obs_np)
    ls_np = rng.uniform(-2.5, -0.5, ACT).astype(np.float32)
    ls = _cuda(ls_np)
    ones = torch.ones(E, dtype=torch.uint8, device="cuda")
    state, mean, lp_mean = _forward(L, eng, pol_struct, mcp, obs, ls, zf.stats, 1, ones, STEP0)
    zref = R.zf_merge(zref, obs_np)
    check_zfilter(zf.stats, state, zref, obs_np, kinds, tag, (obs_np.astype(np.float64) ** 2).sum(0))
    st = state.cpu().numpy()
    mref, scale = ref_fn(st)
    mu = mean.cpu().numpy()
    e_mean = (np.abs(mu - mref) / scale).max()
    assert np.isfinite(mu).all() and e_mean <= MEAN_REL, (tag, e_mean)
    assert np.abs(lp_mean.cpu().numpy() - (-ls_np.astype(np.float64).sum() - ACT * R.LOG_SQRT_2PI)).max() <= LOGP_REL * (np.abs(ls_np).sum() + ACT * R.LOG_SQRT_2PI)
    # frozen statistics, every action sampled: the same mean plus exp(log_std) times the fp64 normal of (row, dim) at STEP0 + 1
    stats_before = zf.stats.clone()
    state2, a, lp = _forward(L, eng, pol_struct, mcp, obs, ls, zf.stats, 0, None, STEP0 + 1)
    assert torch.equal(zf.stats, stats_before) and torch.equal(state2, state)
    eps, _ = R.noise(SEED, STEP0 + 1, E, ACT)
    want = mu.astype(np.float64) + np.exp(ls_np.astype(np.float64)) * eps
    an = a.cpu().numpy()
    e_a = (np.abs(an - want) / (ulp32(want) + np.exp(ls_np) * 2.0 ** -24 * SAMPLE_ULPS * R.TAIL)).max()
    lref, mag = R.gaussian_logp(mu, ls_np, an)
    e_lp = (np.abs(lp.cpu().numpy() - lref) / mag).max()
    assert e_a <= 1.0 and e_lp <= LOGP_REL, (tag, e_a, e_lp)
    return e_mean


@pytest.mark.parametrize("E", [200, 4097])
def test_policy_forward_against_fp64(E, clip, shape_vec):
    """uhc_policy_forward (657-2048-1024-512-105 gelu) and uhc_policy_forward_mcp (P = 1, 3, 8 relu primitives, composer 300-200); E = 4097 leaves
    a partial last 128-row tile"""
    from uhc_b200 import nn
    L = _lib()
    eng = _engine(E, clip)
    rng = np.random.default_rng(E)
    obs = _obs(rng, E, shape_vec)
    out = {}
    try:
        pol = nn.MLPNet(OBS, (2048, 1024, 512), ACT, "gelu", seed=E)
        Ws, bs = _mlp_weights(pol)
        out["mlp"] = check_policy_call(L, eng, nn.mlp_struct(pol), False, lambda s: R.mlp_forward(Ws, bs, s, "gelu"), obs, shape_vec, rng, (E, "mlp"))
        for P in (1, 3, 8):
            net = nn.MCPNet(OBS, (512, 256), ACT, "relu", num_primitive=P, composer_dim=(300, 200), seed=E + P)
            prims = [_mlp_weights(n) for n in net.prims]
            comp = _mlp_weights(net.composer)

            def ref(s):
                m, _, sc = R.mcp_forward(prims, comp, s, "relu")
                return m, sc
            out[f"mcp{P}"] = check_policy_call(L, eng, nn.mcp_struct(net), True, ref, obs, shape_vec, rng, (E, "mcp", P))
    finally:
        eng.close()
    print(f"policy forward E={E}: worst mean error / sum|W||h| " + ", ".join(f"{k} {v:.2e}" for k, v in out.items()))


def test_first_gemm_reads_the_rne_bf16_copy_of_the_state(clip, shape_vec):
    """k_zfilter_apply_bf16's copy, read back through a one-layer policy whose weight rows select single input columns (each output is then one exact
    product): it equals the round-to-nearest-even bf16 of the fp32 state row bit for bit, and the K padding (columns 657..703) reads as zero"""
    import torch
    from uhc_b200 import nn
    L = _lib()
    E = 4097
    eng = _engine(E, clip)
    rng = np.random.default_rng(7)
    obs = _obs(rng, E, shape_vec)
    obs[:, :64] *= 1.0 + 2.0 ** -9 * rng.integers(0, 2, (E, 64))          # plenty of values near bf16 ties
    stats = torch.zeros(1 + 2 * OBS, device="cuda", dtype=torch.float64)
    ls = torch.zeros(ACT, device="cuda")
    ones = torch.ones(E, dtype=torch.uint8, device="cuda")
    try:
        net = nn.MLPNet(OBS, (), ACT, "gelu", seed=0)
        net._prep_bf16()
        Wb = net._bf16_store[0]
        Kp = Wb.shape[1]
        cols = np.arange(Kp)
        got = np.zeros((E, Kp), np.float32)
        state = None
        for c0 in range(0, Kp, ACT):
            sel = cols[c0:c0 + ACT]
            Wb.zero_()
            Wb[torch.arange(len(sel), device="cuda"), _cuda(sel, torch.long)] = 1.0
            net.b[0].zero_()
            st, mean, _ = _forward(L, eng, nn.mlp_struct(net), False, _cuda(obs), ls, stats, int(c0 == 0), ones, STEP0)
            state = st if state is None else state
            got[:, sel] = mean.cpu().numpy()[:, :len(sel)]
        assert np.array_equal(R.bf16_bits(got[:, :OBS]), R.bf16_bits(state.cpu().numpy())), "bf16 copy is not the RNE of the state"
        assert np.array_equal(got[:, :OBS], R.bf16(state.cpu().numpy()))
        assert (got[:, OBS:] == 0).all(), "K padding of the bf16 copy"
    finally:
        eng.close()


def test_rollout_rows_against_fp64(clip):
    """uhc_rollout one row at a time (CUDA graph), obs snapshotted before each row, for noise_rate 0, 0.3, 1 and a rate whose fp32 threshold equals
    one env's uniform draw (that env must sample: u < p, not u <= p).  exps rows and mean-action rows are bit-equal to the numpy Bernoulli draws and
    to the mean; sampled rows are mean + exp(log_std) eps_ref at the device step counter, which advances by one per row from uhc_rollout_set_step;
    the states are the fp64 ZFilter of the snapshots, and after all rows the statistics equal the fp64 merge of every snapshot."""
    import torch
    from uhc_b200 import nn
    from uhc_b200.agent import RolloutBuffer
    L = _lib()
    E, T = 200, 4
    eng = _engine(E, clip, auto_reset=1, t_min=5, t_max=60, reset_seed=11)
    rng = np.random.default_rng(3)
    try:
        eng.reset(clip=np.zeros(E, np.int32), start=rng.integers(0, 40, E).astype(np.int32))
        pol = nn.MLPNet(OBS, (512, 256), ACT, "gelu", seed=5)
        ms = nn.mlp_struct(pol)
        ls_np = rng.uniform(-2.0, -1.0, ACT).astype(np.float32)
        ls = _cuda(ls_np)
        zf = nn.ZFilter(OBS)
        zref, raw2 = R.zf_empty(OBS), np.zeros(OBS)
        u = R.mean_action_uniform(SEED, STEP0, E)
        k_tie = int(np.argmax((u > 0.25) & (u < 0.5)))
        tie_rate = float(np.float32(1.0) - u[k_tie])
        ones = torch.ones(E, dtype=torch.uint8, device="cuda")
        worst, first, same = 0.0, None, None          # same: columns that have held one value in every snapshot so far
        for noise_rate in (0.0, 0.3, 1.0, tie_rate):
            buf = RolloutBuffer(T, E, "cuda")
            assert L.uhc_rollout_set_step(eng.h, C.c_ulonglong(STEP0)) == 0
            for k in range(T):
                snap = eng.obs.clone()
                bs = buf.c_struct(eng.obs)
                rc = L.uhc_rollout(eng.h, C.c_int(1), C.c_int(k), C.byref(ms), _p(ls), _p(zf.stats), C.c_float(R.CLIP), C.c_int(1), C.c_ulonglong(SEED),
                                   C.c_float(noise_rate), C.byref(bs), C.c_int(1), _st())
                assert rc == 0, L.uhc_rollout_last_error()
                torch.cuda.synchronize()
                x = snap.cpu().numpy()
                zref = R.zf_merge(zref, x)
                raw2 += (x.astype(np.float64) ** 2).sum(0)
                first = x[0] if first is None else first
                same = (x == first).all(0) if same is None else same & (x == first).all(0)
                assert same[SHAPE_COLS].all()                         # one subject: the shape vector is constant over every env and step
                kinds = np.where(same, "const", "normal").astype(object)
                check_zfilter(zf.stats, buf.states[k], zref, x, kinds, ("rollout", noise_rate, k), raw2)
                step = STEP0 + k
                flags = R.mean_action_flags(SEED, step, E, noise_rate) if noise_rate < 1.0 else np.zeros(E, np.uint8)
                exps = buf.exps[k].cpu().numpy()
                assert np.array_equal(exps, (1 - flags).astype(np.float32)), (noise_rate, k, np.flatnonzero(exps != 1 - flags)[:10])
                if noise_rate == tie_rate and k == 0:
                    assert flags[k_tie] == 0 and exps[k_tie] == 1.0
                # the mean of this row: the same policy on the same snapshot with the statistics this row normalised with
                frozen = zf.stats.clone()
                _, mean, _ = _forward(L, eng, ms, False, snap, ls, frozen, 0, ones)
                assert torch.equal(frozen, zf.stats)
                mu, a = mean.cpu().numpy(), buf.actions[k].cpu().numpy()
                det = flags == 1
                assert np.array_equal(a[det], mu[det]), (noise_rate, k)
                eps, _ = R.noise(SEED, step, E, ACT)
                want = mu.astype(np.float64) + np.exp(ls_np.astype(np.float64)) * eps
                e_a = (np.abs(a - want) / (ulp32(want) + np.exp(ls_np) * 2.0 ** -24 * SAMPLE_ULPS * R.TAIL))[~det]
                assert e_a.size == 0 or e_a.max() <= 1.0, (noise_rate, k, e_a.max())
                worst = max(worst, e_a.max() if e_a.size else 0.0)
                lref, mag = R.gaussian_logp(mu, ls_np, a)
                assert (np.abs(buf.logp[k].cpu().numpy() - lref) / mag).max() <= LOGP_REL
            got = C.c_ulonglong(0)
            assert L.uhc_rollout_get_step(eng.h, C.byref(got)) == 0 and got.value == STEP0 + T
        n, mean, S = zref
        s = zf.stats.cpu().numpy()
        assert s[0] == n == 4 * T * E
        assert np.abs(s[1:1 + OBS] - mean).max() <= ZF_MEAN_REL * (np.abs(mean) + R.zf_std(zref)).max()
        assert (s[1 + OBS:][SHAPE_COLS] == 0).all()
    finally:
        eng.close()
    print(f"rollout rows: worst sampled action {worst:.2f} of its bound")


# ---------------------------------------------------------------------------------------------------------------- GEMM epilogue
Z_REL = 1e-6             # |z - z_ref| / (sum |x| |w| + |b|), per element  (3.0e-7)
# |y - act(z)| / (2^-24 max(|z|, 1)): the fp32 activation of the kernel's own z  (tanh 1.8, sigmoid 1.4, gelu 3.1; relu and none exact)
Y_F32_ULPS = {"gelu": 10.0, "tanh": 6.0, "sigmoid": 5.0, "relu": 0.0, "none": 0.0}
# fraction of bf16 outputs that are not RNE(act(z)) but its neighbour, where act(z) lies within the fp32 bound of a rounding boundary
# (tanh 1.0e-5, sigmoid 6.7e-6, gelu 1.0e-2: the erf approximation is accurate in absolute terms, so gelu's tiny negative tail, where bf16 is
# fine-grained, flips most)
BF16_FLIPS = {"gelu": 5e-2, "tanh": 3e-5, "sigmoid": 2e-5, "relu": 0.0, "none": 0.0}


@pytest.mark.parametrize("act", ["gelu", "tanh", "relu", "sigmoid", "none"])
def test_gemm_epilogue_one_layer(act):
    """uhc_linear_forward_tc_train: z against the fp64 product of the same bf16 operands (per-element accumulation bound), the fp32 y against the exact
    activation of the kernel's own z, the bf16 y equal to the RNE of that activation but for rare one-ulp flips, and the poisoned padding columns of the
    bf16 buffer (ld = N rounded up to 64) zeroed"""
    import torch
    from uhc_b200 import nn
    L = nn._lib()
    rng = np.random.default_rng(["gelu", "tanh", "relu", "sigmoid", "none"].index(act))
    worst = np.zeros(3)
    for N in (1, 105, 200, 300, 2048):
        for M, K in ((77, 657), (4097, 200), (1000, 64)):
            Kp, ld = (K + 63) // 64 * 64, (N + 63) // 64 * 64
            x = np.zeros((M, Kp), np.float32); x[:, :K] = R.bf16(rng.standard_normal((M, K)).astype(np.float32) * 1.5)
            W = np.zeros((N, Kp), np.float32); W[:, :K] = R.bf16((rng.standard_normal((N, K)) / math.sqrt(K)).astype(np.float32))
            b = rng.standard_normal(N).astype(np.float32)
            ybf = torch.full((M, ld), 7.0, device="cuda", dtype=torch.bfloat16)
            yf = torch.full((M, N), float("nan"), device="cuda")
            z = torch.full((M, N), float("nan"), device="cuda")
            xd, Wd, bd = _cuda(x, torch.bfloat16), _cuda(W, torch.bfloat16), _cuda(b)      # held: a freed operand's memory could be reused before the launch runs
            rc = L.uhc_linear_forward_tc_train(_p(xd), _p(Wd), _p(bd), _p(ybf), _p(yf), _p(z), M, N, Kp, ld, nn.ACT[act], _st())
            assert rc == 0, L.uhc_tc_last_error()
            torch.cuda.synchronize()
            zg, yg = z.cpu().numpy().astype(np.float64), yf.cpu().numpy().astype(np.float64)
            yb = ybf.view(torch.int16).cpu().numpy().view(np.uint16)
            x64, W64 = x.astype(np.float64), W.astype(np.float64)
            zr = x64 @ W64.T + b
            scale = np.abs(x64) @ np.abs(W64).T + np.abs(b)
            e_z = (np.abs(zg - zr) / scale).max()
            ya = R.act(act, zg)
            e_y = (np.abs(yg - ya) / (2.0 ** -24 * np.maximum(np.abs(zg), 1.0))).max()
            # the bf16 output is RNE of the fp32 activation, which may sit anywhere within its bound of act(z): it lies between the roundings of the
            # bound's two ends (rounding is monotone), and equals RNE(act(z)) but for a bounded fraction
            tol = Y_F32_ULPS[act] * 2.0 ** -24 * np.maximum(np.abs(zg), 1.0)
            ybv = R.bf16_value(yb[:, :N]).astype(np.float64)
            lo, hi = R.bf16((ya - tol).astype(np.float32)), R.bf16((ya + tol).astype(np.float32))
            flips = (yb[:, :N] != R.bf16_bits(ya.astype(np.float32))).mean()
            tag = (act, M, N, K)
            assert e_z <= Z_REL, (tag, "z", e_z)
            assert e_y <= Y_F32_ULPS[act], (tag, "fp32 y", e_y)
            assert ((ybv >= lo) & (ybv <= hi)).all() and flips <= BF16_FLIPS[act], (tag, "bf16 y", flips)
            assert (yb[:, N:] == 0).all(), (tag, "padding")
            worst = np.maximum(worst, (e_z, e_y, flips))
    print(f"epilogue {act}: worst z {worst[0]:.2e} of sum|x||w|, fp32 y {worst[1]:.2f} ulps, bf16 flips {worst[2]:.2e}")
