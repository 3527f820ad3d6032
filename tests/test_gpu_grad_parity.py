"""GPU: the PPO update's kernels against the fp64 autograd reference tests/ppo_ref.py (itself pinned to the reference's traces by
tests/test_ppo_ref.py), compared on the GRADIENTS and loss values, before Adam sees them.  Adam's first steps are ~ lr sign(g): a gradient of the
wrong magnitude but the right sign moves the parameters the same way, so the parameter-change tests elsewhere cannot see it.

Every bound sits at least 3x above the worst error measured on an H100 (recorded beside it) and far below what a wrong factor, a wrong row
count, a missing clip or a missing softmax / GELU term produces (0.1 to 1 relative)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import ppo_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _check(name, err, bound):
    print(f"[grad-parity] {name}: {err:.3e} (bound {bound:.1e})")
    assert err < bound, (name, err, bound)


def _lib():
    from uhc_b200 import nn
    return nn._lib()


def _st():
    from uhc_b200 import nn
    return nn._stream(torch.zeros(1, device=DEV))


def _p(t):
    from uhc_b200 import nn
    return nn._p(t)


def _maxrel(got, ref):
    """max |got - ref| over max |ref| (element-wise agreement at the tensor's scale)"""
    got, ref = got.double(), ref.double()
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


def _tensor_metrics(got, ref):
    """(relative Frobenius error, 1 - cosine, |norm ratio - 1|)"""
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    rn, gn = ref.norm(), got.norm()
    return float((got - ref).norm() / rn), float(1.0 - (got @ ref) / (gn * rn)), float(abs(gn / rn - 1.0))


# ------------------------------------------------------------------------------------------------ loss heads and sampling
def _policy_grad_case(M, A, seed, exps_kind="mixed"):
    """inputs whose ratios are placed on purpose: exactly 1, inside (1 - eps, 1 + eps), below and above the clip interval, ON its edges; with
    advantages > 0, < 0 and == 0"""
    from uhc_b200 import nn
    g = torch.Generator().manual_seed(seed)
    log_std = torch.linspace(-3.0, 0.5, A, dtype=torch.float64)[torch.randperm(A, generator=g)]
    mean = torch.randn(M, A, generator=g, dtype=torch.float64)
    actions = mean + torch.exp(log_std) * torch.randn(M, A, generator=g, dtype=torch.float64)
    f32 = lambda t: t.float().to(DEV).contiguous()
    mean32, ls32, act32 = f32(mean), f32(log_std), f32(actions)
    lp = nn.gaussian_logprob(mean32, ls32, act32)                  # the kernel's own log-probabilities: ratio targets are exact for it
    eps = 0.2
    targets = torch.tensor([1.0, 1.0, 0.93, 1.12, 1.05, 0.5, 0.7, 1.3, 2.5, 1.0 - eps, 1.0 + eps], dtype=torch.float64)
    ratio_t = targets[torch.randint(0, len(targets), (M,), generator=g)]
    fixed = lp.double().cpu() - torch.log(ratio_t)
    adv = torch.tensor([1.3, -0.7, 0.0], dtype=torch.float64)[torch.randint(0, 3, (M,), generator=g)] * torch.rand(M, generator=g, dtype=torch.float64).add(0.5)
    if exps_kind == "mixed":
        exps = (torch.rand(M, generator=g) > 0.25).double()
        exps[0] = 1.0
    elif exps_kind == "zero":
        exps = torch.zeros(M, dtype=torch.float64)
    else:
        exps = torch.ones(M, dtype=torch.float64)
    return dict(mean=mean32, log_std=ls32, actions=act32, adv=f32(adv), fixed=f32(fixed), exps=f32(exps), eps=eps)


def _policy_grad_kernels(c, M, A):
    L, st = _lib(), _st()
    count = float((c["exps"] != 0).sum())
    out = []
    for dev_count in (False, True):
        dmean = torch.full((M, A), 7.0, device=DEV)
        loss = torch.zeros(1, device=DEV)
        if dev_count:
            inv = torch.tensor([1.0 / max(count, 1.0)], device=DEV)
            rc = L.uhc_ppo_policy_grad_dev(_p(c["mean"]), _p(c["log_std"]), _p(c["actions"]), _p(c["adv"]), _p(c["fixed"]), _p(c["exps"]), C.c_float(c["eps"]),
                                           _p(inv), _p(dmean), _p(loss), M, A, st)
        else:
            rc = L.uhc_ppo_policy_grad(_p(c["mean"]), _p(c["log_std"]), _p(c["actions"]), _p(c["adv"]), _p(c["fixed"]), _p(c["exps"]), C.c_float(c["eps"]),
                                       C.c_float(1.0 / max(count, 1.0)), _p(dmean), _p(loss), M, A, st)
        assert rc == 0
        out.append((dmean, loss))
    torch.cuda.synchronize()
    return out


def test_policy_gradient_matches_fp64_autograd():
    worst_g, worst_l = 0.0, 0.0
    for M in (1, 7, 8, 8193):
        for A in (1, 31, 32, 33, 75, 105, 315):
            c = _policy_grad_case(M, A, seed=M * 1000 + A)
            (d_host, l_host), (d_dev, l_dev) = _policy_grad_kernels(c, M, A)
            # the two entry points differ only in where 1/count lives (the loss is a float atomic sum: its order may differ)
            assert torch.equal(d_host, d_dev) and abs(l_host.item() - l_dev.item()) <= 1e-5 * max(abs(l_host.item()), 1e-3), (M, A)
            mean = c["mean"].double().cpu().requires_grad_(True)
            ls, a, fixed, adv, exps = (c[k].double().cpu() for k in ("log_std", "actions", "fixed", "adv", "exps"))
            logp = R.gaussian_logp(mean, ls, a)
            loss = R.surrogate_loss(logp, fixed, adv, exps, c["eps"])
            (dref,) = torch.autograd.grad(loss, mean)
            ratio = torch.exp(logp.detach() - fixed)
            # the gradient every selected row would have without the clip: its largest entry is the scale of the comparison
            sel = (exps != 0).double()
            unclipped = (-ratio * adv * sel / max(float(sel.sum()), 1.0))[:, None] * (a - mean.detach()) * torch.exp(-2 * ls)
            scale = unclipped.abs().max().clamp_min(1e-30)
            # rows within 1e-4 of a clip edge (the fp32 and fp64 ratios differ by up to ~|logp| 1e-7): either one-sided gradient is right
            edge = ((ratio - (1 - c["eps"])).abs() < 1e-4) | ((ratio - (1 + c["eps"])).abs() < 1e-4)
            got = d_host.double().cpu()
            inner = ~edge
            err = float((got[inner] - dref[inner]).abs().max() / scale) if inner.any() else 0.0
            worst_g = max(worst_g, err)
            if edge.any():
                e_clip, e_unclip = got[edge].abs().amax(1), (got[edge] - unclipped[edge]).abs().amax(1)
                assert (torch.minimum(e_clip, e_unclip) <= 3e-5 * scale).all(), (M, A)
            lerr = abs(l_host.item() - loss.item()) / max(abs(loss.item()), 1e-3)
            worst_l = max(worst_l, lerr)
            assert torch.isfinite(got).all() and ((exps == 0)[:, None].expand(-1, A) <= (got == 0)).all(), (M, A)   # unselected rows: zero gradient
    _check("policy dmean, max |err| / max |unclipped dmean|", worst_g, 3e-5)      # measured 8.4e-6
    _check("policy surrogate loss, relative", worst_l, 2e-5)                         # measured 4.7e-6


def test_policy_gradient_with_no_selected_row_is_zero():
    for M, A in ((7, 33), (8193, 105)):
        c = _policy_grad_case(M, A, seed=5, exps_kind="zero")
        for dmean, loss in _policy_grad_kernels(c, M, A):
            assert torch.isfinite(dmean).all() and (dmean == 0).all() and loss.item() == 0.0


@pytest.mark.parametrize("M", [1, 1000, 131072])
def test_value_gradient_and_loss(M):
    L, st = _lib(), _st()
    g = torch.Generator().manual_seed(M)
    v64, r64 = torch.randn(M, generator=g, dtype=torch.float64), torch.randn(M, generator=g, dtype=torch.float64) * 2 + 0.5
    v, r = v64.float().to(DEV), r64.float().to(DEV)
    for M_total in (M, 3 * M + 5):
        dv, loss = torch.empty(M, device=DEV), torch.zeros(1, device=DEV)
        if M_total == M:
            assert L.uhc_value_grad(_p(v), _p(r), _p(dv), _p(loss), M, st) == 0
        else:
            assert L.uhc_value_grad_n(_p(v), _p(r), _p(dv), _p(loss), M, C.c_long(M_total), st) == 0
        torch.cuda.synchronize()
        vl = v.double().cpu().requires_grad_(True)
        ref = R.value_loss(vl, r.double().cpu()) * (M / M_total)      # this shard's share of the global batch's mean
        (dref,) = torch.autograd.grad(ref, vl)
        # measured 7.2e-8 (dv), 1.6e-6 (the loss: a float atomic sum over up to 131072 rows)
        _check(f"value dv M={M} M_total={M_total}", _maxrel(dv.cpu(), dref), 3e-7)
        _check(f"value loss M={M} M_total={M_total}", abs(loss.item() - ref.item()) / ref.item(), 1e-5)


@pytest.mark.parametrize("A", [105, 315])
def test_gaussian_logprob_and_sample(A):
    from uhc_b200 import nn
    M = 1000
    g = torch.Generator().manual_seed(A)
    ls = torch.linspace(-3.0, 0.5, A, dtype=torch.float64)[torch.randperm(A, generator=g)]
    mean = torch.randn(M, A, generator=g, dtype=torch.float64).float().double()
    act = (mean + torch.exp(ls) * torch.randn(M, A, generator=g, dtype=torch.float64)).float().double()
    ls = ls.float().double()
    f = lambda t: t.float().to(DEV).contiguous()
    lp = nn.gaussian_logprob(f(mean), f(ls), f(act)).double().cpu()
    ref = R.gaussian_logp(mean, ls, act)
    # the per-row fp32 sum of A terms of size ~1: the bound scales with the row's sum of absolute terms
    terms = ((act - mean) ** 2 / (2 * torch.exp(2 * ls)) + ls.abs() + 0.92).sum(1)
    _check(f"logprob A={A}, |err| / sum |terms|", float(((lp - ref).abs() / terms).max()), 1e-7)           # measured 2.0e-8
    det = (torch.arange(M) % 3 == 0).to(torch.uint8)
    a, lps = nn.gaussian_sample(f(mean), f(ls), seed=7, step=3, mean_action=det.to(DEV))
    a, lps = a.double().cpu(), lps.double().cpu()
    assert torch.equal(a[det.bool()], mean[det.bool()])
    ref_s = R.gaussian_logp(mean, ls, a)
    terms = ((a - mean) ** 2 / (2 * torch.exp(2 * ls)) + ls.abs() + 0.92).sum(1)
    _check(f"sample logp A={A}, |err| / sum |terms|", float(((lps - ref_s).abs() / terms).max()), 1e-7)     # measured 2.2e-8


# ------------------------------------------------------------------------------------------------ advantages, normalisation, clip, Adam
@pytest.mark.parametrize("E", [1, 127, 129, 4096])
@pytest.mark.parametrize("T", [1, 8, 64])
def test_gae_lock_step(T, E):
    L, st = _lib(), _st()
    g = torch.Generator().manual_seed(T * 10000 + E)
    r = torch.rand(T, E, generator=g, dtype=torch.float64).float().double()
    v = torch.randn(T, E, generator=g, dtype=torch.float64).float().double()
    m = (torch.rand(T, E, generator=g) > 0.1).double()
    m[-1, ::3] = 0.0                                                # terminal rows at the end of the rollout
    last = torch.randn(E, generator=g, dtype=torch.float64).float().double()
    f = lambda t: t.float().to(DEV).contiguous()
    for with_last in (False, True):
        adv, ret = torch.empty(T, E, device=DEV), torch.empty(T, E, device=DEV)
        lv = f(last) if with_last else None
        assert L.uhc_gae(_p(f(r)), _p(f(m)), _p(f(v)), _p(lv), C.c_float(0.95), C.c_float(0.95), _p(adv), _p(ret), T, E, st) == 0
        torch.cuda.synchronize()
        a_ref, r_ref = R.gae_te(r, m, v, 0.95, 0.95, last if with_last else None)
        _check(f"gae adv T={T} E={E} last={with_last}", _maxrel(adv.cpu(), a_ref), 2e-6)      # measured 3.2e-7
        _check(f"gae ret T={T} E={E} last={with_last}", _maxrel(ret.cpu(), r_ref), 2e-6)      # measured 4.2e-7


@pytest.mark.parametrize("n,offset", [(2, 0.0), (1000, 0.0), (100003, 0.0), (100003, 1e3)])
def test_advantage_normalisation(n, offset):
    L, st = _lib(), _st()
    g = torch.Generator().manual_seed(n)
    x = (torch.randn(n, generator=g, dtype=torch.float64) * 1.7 + offset).float()
    ref = R.normalize(x.double())
    a = x.to(DEV).clone()
    scratch = torch.zeros(2, device=DEV, dtype=torch.float64)
    assert L.uhc_normalize_advantages(_p(a), C.c_long(n), _p(scratch), st) == 0
    # the sharded pair: local moments of two shards, summed (the all-reduce), each shard normalised with the global count read from the device
    k = n // 2
    sh = [x[:k].to(DEV).clone(), x[k:].to(DEV).clone()]
    moms = [torch.zeros(2, device=DEV, dtype=torch.float64) for _ in sh]
    for s, mo in zip(sh, moms):
        if s.numel():
            assert L.uhc_adv_moments(_p(s), C.c_long(s.numel()), _p(mo), st) == 0
    tot = moms[0] + moms[1]
    ntot = torch.tensor([float(n)], device=DEV, dtype=torch.float64)
    for s in sh:
        if s.numel():
            assert L.uhc_adv_normalize(_p(s), C.c_long(s.numel()), _p(tot), _p(ntot), st) == 0
    torch.cuda.synchronize()
    # fp32 output: the bound is a few fp32 ulps of the input's magnitude over the std (offset 1e3: the mean itself is rounded to fp32)
    bound = 2e-6 if offset == 0.0 else 6e-5          # measured 4.2e-7 and 1.5e-5
    _check(f"normalize n={n} offset={offset}", float((a.double().cpu() - ref).abs().max()), bound)
    _check(f"sharded normalize n={n} offset={offset}", float((torch.cat(sh).double().cpu() - ref).abs().max()), bound)


def _adam_case(n, step0, clip, seed):
    """p, g (fp32), resumed Adam state at step0 (zeros when step0 = 0) and max_norm for the clip mode"""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g).float() * 0.05
    grads = [(torch.randn(n, generator=g) * torch.exp(torch.randn(n, generator=g) * 2) * 0.01).float() for _ in range(3)]
    m = (torch.randn(n, generator=g) * 0.01).float() if step0 else torch.zeros(n)
    v = (m.double() ** 2 * 2 + 1e-6 * torch.rand(n, generator=g, dtype=torch.float64)).float() if step0 else torch.zeros(n)
    norm = float(grads[0].double().norm())
    max_norm = {"off": None, "active": 0.3 * norm, "edge": norm}[clip]
    return p, grads, m, v, max_norm


@pytest.mark.parametrize("n", [1000, 1056 * 256 + 777])
@pytest.mark.parametrize("steps,step0", [(1, 0), (2, 0), (10, 0), (2, 10000)])
@pytest.mark.parametrize("clip", ["off", "active", "edge"])
def test_adam_with_clip_matches_torch(n, steps, step0, clip):
    """uhc_sqsum + uhc_adam_step against fp64 clip_grad_norm_ + torch.optim.Adam fed the same fp32 gradients (the clip on every step here)"""
    L, st = _lib(), _st()
    lr = 1e-3
    p, grads, m, v, max_norm = _adam_case(n, step0, clip, seed=n + steps + step0)
    pd, md, vd = p.to(DEV).clone(), m.to(DEV).clone(), v.to(DEV).clone()
    sq = torch.zeros(1, device=DEV, dtype=torch.float64)
    ref = p.double().clone().requires_grad_(True)
    opt = R.adam([ref], lr)
    if step0:
        opt.state[ref] = {"step": torch.tensor(float(step0)), "exp_avg": m.double().clone(), "exp_avg_sq": v.double().clone()}
    for s in range(steps):
        gr = grads[s % len(grads)]
        gd = gr.to(DEV)
        if max_norm is not None:
            sq.zero_()
            assert L.uhc_sqsum(_p(gd), C.c_long(n), _p(sq), st) == 0
        assert L.uhc_adam_step(_p(pd), _p(gd), _p(md), _p(vd), C.c_long(n), C.c_float(lr), C.c_float(0.9), C.c_float(0.999), C.c_float(1e-8), step0 + s + 1,
                               _p(sq) if max_norm is not None else None, C.c_float(max_norm or 0.0), st) == 0
        ref.grad = gr.double().clone()
        if max_norm is not None:
            torch.nn.utils.clip_grad_norm_([ref], max_norm)
        opt.step()
        if max_norm is not None and s == 0:
            torch.cuda.synchronize()
            _check(f"sqsum n={n}", abs(sq.item() - float((gr.double() ** 2).sum())) / float((gr.double() ** 2).sum()), 1e-13)     # measured 1.9e-15
    torch.cuda.synchronize()
    d_got, d_ref = pd.double().cpu() - p.double(), ref.detach() - p.double()
    _check(f"adam n={n} steps={steps} from={step0} clip={clip}, max |err| / lr", float((d_got - d_ref).abs().max()) / lr, 3e-4)   # measured 5.8e-5
    # the C ABI takes the betas as floats: 1 - 0.999f = 9.99987e-4, so the second moment sits 1.29e-5 below fp64's (measured 1.31e-5)
    _check(f"adam moments n={n} steps={steps} from={step0} clip={clip}", max(_maxrel(md.cpu(), opt.state[ref]["exp_avg"]), _maxrel(vd.cpu(), opt.state[ref]["exp_avg_sq"])), 5e-5)


# ------------------------------------------------------------------------------------------------ MLP backward and the mixture head
def _mlp_case(D, hs, A, htype, M, seed):
    from uhc_b200 import nn
    net = nn.MLPNet(D, hs, A, htype, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(M, D, generator=g).clamp(-5, 5).to(DEV)
    dy = (torch.randn(M, A, generator=g) * 0.01).to(DEV)
    return net, x, dy


def _mlp_ref_grads(net, x, dy, bf16):
    """fp64 autograd of sum(mlp(x) * dy) wrt [W0, b0, ...] and x; bf16: the weights, the input and the stored hidden activations rounded as the
    tensor-core path rounds them (without the activation rounding a relu unit whose pre-activation is within bf16 noise of 0 flips its mask)"""
    rnd = (lambda t: t.bfloat16().double()) if bf16 else (lambda t: t.double())
    params = [rnd(p) if i % 2 == 0 else p.double() for i, p in enumerate(net.params())]
    params = [p.detach().clone().requires_grad_(True) for p in params]
    xr = rnd(x).detach().clone().requires_grad_(True)
    out = R.mlp(params, xr, net.htype, store=R.bf16_store if bf16 else None)
    gr = torch.autograd.grad((out * dy.double()).sum(), params + [xr])
    return gr[:-1], gr[-1]


@pytest.mark.parametrize("htype", ["gelu", "tanh", "relu", "sigmoid"])
@pytest.mark.parametrize("M", [1, 77, 8193])
def test_fp32_mlp_backward_matches_fp64_autograd(htype, M):
    from uhc_b200 import nn
    net, x, dy = _mlp_case(657, (130, 66), 105, htype, M, seed=M)
    y, ctx = net.forward(x, save=True)
    grads = net.backward(dy, ctx)
    dx = torch.empty_like(x)                                          # the input layer's dX (MLPNet.backward stops at the first layer's weights)
    assert _lib().uhc_linear_backward(_p(x), _p(net.W[0]), _p(_first_layer_dz(net, x, dy)), _p(dx), _p(torch.empty_like(net.W[0])),
                                      _p(torch.empty_like(net.b[0])), M, net.W[0].shape[0], 657, nn._stream(x)) == 0
    torch.cuda.synchronize()
    ref, dx_ref = _mlp_ref_grads(net, x, dy, bf16=False)
    worst = max(_tensor_metrics(g, r)[0] for g, r in zip(grads, ref))
    _check(f"fp32 backward {htype} M={M}, worst relative Frobenius error", worst, 1e-5)     # measured 1.7e-6
    _check(f"fp32 backward {htype} M={M}, dX", _tensor_metrics(dx, dx_ref)[0], 3e-6)        # measured 5.3e-7


def _first_layer_dz(net, x, dy):
    """dz of the first layer, from the fp32 kernels (uhc_linear_backward of the layers above, uhc_act_backward)"""
    from uhc_b200 import nn
    y, (saved, zs) = net.forward(x, save=True)
    dz = dy.contiguous()
    L = _lib()
    for i in range(len(net.W) - 1, 0, -1):
        M, K = saved[i].shape
        dx = torch.empty(M, K, device=DEV)
        assert L.uhc_linear_backward(_p(saved[i]), _p(net.W[i]), _p(dz), _p(dx), _p(torch.empty_like(net.W[i])), _p(torch.empty_like(net.b[i])), M, net.W[i].shape[0], K,
                                     nn._stream(x)) == 0
        assert L.uhc_act_backward(_p(dx), _p(zs[i - 1]), _p(dx), C.c_long(dx.numel()), nn.ACT[net.htype], nn._stream(x)) == 0
        dz = dx
    return dz


@pytest.mark.parametrize("hs,htype", [((256, 128), "gelu"), ((256, 128), "tanh"), ((130, 66), "gelu"), ((130, 66), "relu"), ((128, 64), "sigmoid")])
@pytest.mark.parametrize("M", [77, 8193])
def test_tensor_core_backward_matches_fp64_autograd(hs, htype, M):
    """TCTrainer: bf16 operands, fp32 accumulation; fused dX + activation backward where K % 4 == 0, the scalar k_dact_bf16 where N % 4 != 0"""
    from uhc_b200 import nn
    net, x, dy = _mlp_case(657, hs, 105, htype, M, seed=M + len(htype))
    tr = nn.TCTrainer(net)
    xb, xT = tr.prepare_input(x)
    _, ctx = tr.forward(xb)
    tr.backward(dy, ctx, xT)
    torch.cuda.synchronize()
    ref, _ = _mlp_ref_grads(net, x, dy, bf16=True)
    worst = [0.0, 0.0, 0.0]
    for i, (g, r) in enumerate(zip(net.grad_views(), ref)):
        m = _tensor_metrics(g, r)
        worst = [max(a, b) for a, b in zip(worst, m)]
    # measured 3.1e-3, 4.8e-6, 8.4e-4 (every tensor of every case)
    _check(f"tc backward {hs} {htype} M={M}, relative Frobenius", worst[0], 1e-2)
    _check(f"tc backward {hs} {htype} M={M}, 1 - cosine", worst[1], 3e-5)
    _check(f"tc backward {hs} {htype} M={M}, |norm ratio - 1|", worst[2], 3e-3)


@pytest.mark.parametrize("P", [1, 4, 8, 16])
@pytest.mark.parametrize("A", [75, 105])
def test_mixture_head_forward_and_backward(P, A):
    L, st = _lib(), _st()
    M = 1001
    g = torch.Generator().manual_seed(P * 100 + A)
    xall = torch.randn(P, M, A, generator=g).float()
    c = torch.randn(M, P, generator=g).float() * 2
    c[::7] *= 40.0                                                   # logits of magnitude ~80: softmax must subtract the row maximum
    dmean = torch.randn(M, A, generator=g).float()
    xd, cd, dmd = xall.to(DEV), c.to(DEV), dmean.to(DEV)
    mean, w = torch.empty(M, A, device=DEV), torch.empty(M, P, device=DEV)
    dxall, dc = torch.empty(P, M, A, device=DEV), torch.empty(M, P, device=DEV)
    assert L.uhc_mcp_combine(_p(xd), _p(cd), _p(w), _p(mean), M, A, P, st) == 0
    assert L.uhc_mcp_backward(_p(xd), _p(w), _p(dmd), _p(dxall), _p(dc), M, A, P, st) == 0
    torch.cuda.synchronize()
    x64, c64 = xall.double().requires_grad_(True), c.double().requires_grad_(True)
    m_ref, w_ref = R.mix(x64, c64)
    gx, gc = torch.autograd.grad((m_ref * dmean.double()).sum(), [x64, c64])
    assert torch.isfinite(mean).all() and torch.isfinite(dc).all()
    # measured 2.5e-7, 2.3e-7, 1.4e-7, 6.2e-7 (dc)
    _check(f"mcp mean P={P} A={A}", _maxrel(mean.cpu(), m_ref.detach()), 1e-6)
    _check(f"mcp weight P={P} A={A}", float((w.cpu().double() - w_ref.detach()).abs().max()), 1e-6)
    _check(f"mcp dxall P={P} A={A}", _maxrel(dxall.cpu(), gx), 1e-6)
    if P > 1:
        # dc rows: |dc| ~ w (dw - w.dw); the error is relative to the row's sum |w_k dw_k|
        rs = (w_ref.detach() * (xall.double() * dmean.double()).sum(-1).t().abs()).sum(1, keepdim=True) + 1e-30
        _check(f"mcp dc P={P} A={A}, |err| / row scale", float(((dc.cpu().double() - gc).abs() / rs).max()), 3e-6)
    else:
        assert (dc == 0).all()


def test_mixture_head_rejects_17_primitives():
    L, st = _lib(), _st()
    z = torch.zeros(17 * 8 * 4, device=DEV)
    assert L.uhc_mcp_combine(_p(z), _p(z), _p(z), _p(z), 8, 4, 17, st) == -2
    assert L.uhc_mcp_backward(_p(z), _p(z), _p(z), _p(z), _p(z), 8, 4, 17, st) == -2


# ------------------------------------------------------------------------------------------------ the whole update, on its gradients
def _bf16_params(net):
    return [(p.bfloat16().double() if i % 2 == 0 else p.double()).detach().clone().requires_grad_(True) for i, p in enumerate(net.params())]


def _grad_views(net):
    return [net.gflat[o:o + n].view_as(p) for (o, n), p in zip(net._offs, net.params())]


def _update_case(kind):
    """(policy, value, states, actions, returns, advantages, exps, log_std)"""
    from uhc_b200 import nn
    if kind == "mcp":
        import os
        z = np.load(os.path.join(os.path.dirname(__file__), "golden", "mcp_ppo.npz"))
        hs, P, cd = tuple(int(h) for h in z["hsize"]), int(z["nprim"]), tuple(int(h) for h in z["composer_dim"])
        S, A = z["states"].shape[1], z["actions"].shape[1]
        pol = nn.MCPNet(S, hs, A, "relu", num_primitive=P, composer_dim=cd, device=DEV, seed=1)
        pol.load_state_dict({k[3:]: z[k] for k in z.files if k.startswith("p0.")})
        val = nn.MLPNet(S, hs, 1, "relu", device=DEV, head_name="value_head", seed=2)
        val.load_state_dict({k[3:]: z[k] for k in z.files if k.startswith("v0.")})
        f = lambda k: torch.tensor(np.asarray(z[k], dtype=np.float32).reshape(z[k].shape[0], -1), device=DEV).squeeze(-1).contiguous() if z[k].ndim > 1 and z[k].shape[1] == 1 \
            else torch.tensor(np.asarray(z[k], dtype=np.float32), device=DEV).contiguous()
        return pol, val, f("states"), f("actions"), f("returns"), f("advantages"), f("exps"), torch.full((A,), -2.3, device=DEV)
    hs, M = {"small": ((256, 128), 2000), "production": ((2048, 1024, 512), 8192)}[kind]
    D, A = 657, 105
    pol = nn.MLPNet(D, hs, A, "gelu", device=DEV, head_name="action_mean", seed=21)
    val = nn.MLPNet(D, hs, 1, "gelu", device=DEV, head_name="value_head", seed=22)
    g = torch.Generator().manual_seed(23)
    states = torch.randn(M, D, generator=g).clamp(-5, 5)
    actions = torch.randn(M, A, generator=g) * 0.1
    returns = torch.randn(M, generator=g) + 0.5
    adv = torch.randn(M, generator=g)
    exps = (torch.rand(M, generator=g) > 0.1).float()
    log_std = torch.linspace(-2.5, -1.5, A)
    return pol, val, *(t.to(DEV).contiguous() for t in (states, actions, returns, adv, exps, log_std))


@pytest.mark.parametrize("kind", ["small", "production", "mcp"])
def test_update_policy_gradients_losses_and_step(kind):
    """uhc_ppo_update_policy with one epoch: both nets' gradients at the initial weights stay in the flat gradient tensors (Adam only reads them).
    They, the two losses and the parameter change are compared with fp64 autograd on the same bf16-rounded weights and states."""
    from uhc_b200 import nn
    pol, val, states, actions, returns, adv, exps, log_std = _update_case(kind)
    lr_p, lr_v = 5e-5, 3e-4
    opt_p, opt_v = nn.Adam(pol.params(), lr_p, net=pol), nn.Adam(val.params(), lr_v, net=val)
    M = states.shape[0]
    p0, v0 = pol.flat.clone(), val.flat.clone()
    # the fp64 reference at the initial weights on the same bf16-rounded weights, states and stored activations, on the GPU (the production net is ~1e11 flops)
    pp, vp = _bf16_params(pol), _bf16_params(val)
    xs = states.bfloat16().double()
    ls, act64, ret64, adv64, ex64 = log_std.double(), actions.double(), returns.double(), adv.double(), exps.double()
    if kind == "mcp":
        n = len(pol.prims[0].params())
        pmean = lambda p, x: R.mcp([p[k * n:(k + 1) * n] for k in range(pol.num_primitive)], p[pol.num_primitive * n:], x, "relu", store=R.bf16_store)[0]
    else:
        pmean = lambda p, x: R.mlp(p, x, pol.htype, store=R.bf16_store)
    logp = R.gaussian_logp(pmean(pp, xs), ls, act64)
    lp_ref = R.surrogate_loss(logp, logp.detach(), adv64, ex64, 0.2)      # epoch 0: fixed log-probs from the same weights, every ratio 1
    gp_ref = R.grads_of(lp_ref, pp)
    lv_ref = R.value_loss(R.mlp(vp, xs, val.htype, store=R.bf16_store), ret64)
    gv_ref = R.grads_of(lv_ref, vp)
    clip = 0.25 * float(torch.sqrt(sum((x ** 2).sum() for x in gp_ref)))   # active: the first policy step is clipped
    tr = nn.CPpoTrainer(pol, val, opt_p, opt_v, M, 1, torch.device(DEV))
    losses = torch.zeros(2, device=DEV)
    tr.update_policy(states, actions, returns, adv, exps, log_std, 0.2, 1, clip, losses)
    torch.cuda.synchronize()
    tr.close()
    for name, net, ref in (("policy", pol, gp_ref), ("value", val, gv_ref)):
        worst = [0.0, 0.0, 0.0]
        for g, r in zip(_grad_views(net), ref):
            worst = [max(a, b) for a, b in zip(worst, _tensor_metrics(g, r))]
        # measured over the three cases: 3.3e-3, 5.5e-6, 8.7e-4
        _check(f"update {kind} {name} gradients, relative Frobenius", worst[0], 1e-2)
        _check(f"update {kind} {name} gradients, 1 - cosine", worst[1], 3e-5)
        _check(f"update {kind} {name} gradients, |norm ratio - 1|", worst[2], 3e-3)
    # (-mean of the selected advantages: the error is relative to their mean magnitude)
    _check(f"update {kind} surrogate loss, relative", abs(losses[0].item() - lp_ref.item()) / float(adv64[ex64 != 0].abs().mean()), 1e-6)  # measured 2.2e-8
    _check(f"update {kind} value loss, relative", abs(losses[1].item() - lv_ref.item()) / lv_ref.item(), 2e-6)                                # measured 3.0e-7
    # the parameter change: p0 + one fp64 Adam step (with the first-step clip) on the gradients the kernels left behind
    for name, net, w0, g, lr, mn in (("policy", pol, p0, pol.gflat, lr_p, clip), ("value", val, v0, val.gflat, lr_v, None)):
        ref = w0.double().clone().requires_grad_(True)
        ref.grad = g.double().clone()
        if mn is not None:
            torch.nn.utils.clip_grad_norm_([ref], mn)
        R.adam([ref], lr).step()
        _check(f"update {kind} {name} step, max |err| / lr", float((net.flat.double() - ref.detach()).abs().max()) / lr, 5e-4)     # measured 1.5e-4


@pytest.mark.parametrize("T,E", [(8, 256), (5, 129)])
def test_full_update_advantages_and_returns(T, E):
    """uhc_ppo_update: GAE over the [T][E] rollout with the V(s_T) bootstrap and the advantage normalisation, against fp64 on the V(s) / V(s_T)
    the tensor-core forward (the same GEMM) gives for the initial value net"""
    from uhc_b200 import nn
    D, A, M = 657, 105, T * E
    pol = nn.MLPNet(D, (256, 128), A, "gelu", device=DEV, head_name="action_mean", seed=31)
    val = nn.MLPNet(D, (256, 128), 1, "gelu", device=DEV, head_name="value_head", seed=32)
    g = torch.Generator().manual_seed(33)
    f = lambda *s: torch.randn(*s, generator=g).to(DEV)
    states, last_states, actions = f(M, D).clamp(-5, 5), f(E, D).clamp(-5, 5), 0.1 * f(M, A)
    rewards = torch.rand(T, E, generator=g).to(DEV)
    masks = (torch.rand(T, E, generator=g) > 0.1).float().to(DEV)
    masks[-1, ::4] = 0.0
    exps = (torch.rand(M, generator=g) > 0.1).float().to(DEV)
    v_s = val.forward_tc(states).reshape(T, E).double().clone()
    v_last = val.forward_tc(last_states).reshape(E).double().clone()
    a_raw, r_ref = R.gae_te(rewards.double(), masks.double(), v_s, 0.95, 0.95, v_last)
    a_ref = R.normalize(a_raw)
    tr = nn.CPpoTrainer(pol, val, nn.Adam(pol.params(), 5e-5, net=pol), nn.Adam(val.params(), 3e-4, net=val), M, E, torch.device(DEV))
    tr.update(states, last_states, actions, rewards, masks, exps, torch.full((A,), -2.3, device=DEV), T, E, 0.95, 0.95, 0.2, 1, 40.0, torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
    adv = tr.advantages(M).double()
    ret = torch.empty(M, device=DEV)
    C.cdll.LoadLibrary("libcudart.so").cudaMemcpy(C.c_void_p(ret.data_ptr()), C.c_void_p(tr.L.uhc_ppo_returns(tr.h)), C.c_size_t(4 * M), C.c_int(3))
    tr.close()
    _check(f"full update advantages T={T} E={E}", float((adv - a_ref.reshape(-1)).abs().max()), 3e-6)      # measured 5.9e-7
    _check(f"full update returns T={T} E={E}", _maxrel(ret, r_ref.reshape(-1)), 1e-6)                     # measured 1.5e-7
