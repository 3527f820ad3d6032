"""GPU: the multi-rank PPO update (world > 1) against fp64 on one GPU, through the in-process all-reduce of tests/loopback_comm.py.

W ranks are W host threads, each with its own stream, trainer and replica of the nets; the trainers call the loopback collective
(uhc_ppo_trainer_set_all_reduce) where a training job calls ncclAllReduce.  The fp64 reference is built for the UNION of the ranks' batches:
GAE over each rank's [T][E] columns on the V(s) / V(s_T) of the tensor-core forward (as tests/test_gpu_grad_parity.py's
test_full_update_advantages_and_returns), the advantage normalisation over the union, fp64 autograd of the union's losses
(tests/ppo_ref.py), the ZFilter's Chan merge over every batch every rank has seen (tests/policy_ref.py).

What is only run with world > 1: the statistics tail (k_stats_pack / k_stats_join / k_zfilter_from_sums in ppo_update.cu, split_double /
join_double in the Python path), the value gradient's 1 / (M world) scale, the global advantage normalisation and selected-row count, and the
ordering of the collectives.  Every bound sits at least 3x above the worst error measured on an H100 SXM (700 W power limit), recorded beside it.
"""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from tests import policy_ref as P
from tests import ppo_ref as R
from tests.loopback_comm import ERR_COUNTS, ERR_EXCEPTION, ERR_REFUSED, NCCL_FLOAT32, NCCL_SUM, LoopbackGradComm, LoopbackGroup

pytestmark = pytest.mark.gpu

DEV = "cuda"
LR_P, LR_V, GAMMA, TAU, EPS = 5e-5, 3e-4, 0.95, 0.95, 0.2

# nets and per-rank rollout shapes.  "v3" / "v3s": obs v3 widths (10 future frames without the shape vector, 5 with it)
KINDS = {
    "small": dict(D=657, A=105, hs=(256, 128), htype="gelu", T=8, E=250),
    "production": dict(D=657, A=105, hs=(2048, 1024, 512), htype="gelu", T=8, E=1024),
    "mcp": dict(D=160, A=75, hs=(256, 128), htype="relu", T=4, E=128, P=4, cd=(64, 32)),
    "v3": dict(D=6400, A=105, hs=(128, 64), htype="gelu", T=4, E=64),
    "v3s": dict(D=3285, A=105, hs=(128, 64), htype="gelu", T=4, E=64),
}


def _check(name, err, bound):
    print(f"[multirank] {name}: {err:.3e} (bound {bound:.1e})")
    assert err < bound, (name, err, bound)


def _tensor_metrics(got, ref):
    """(relative Frobenius error, 1 - cosine, |norm ratio - 1|)"""
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    rn, gn = ref.norm(), got.norm()
    return float((got - ref).norm() / rn), float(1.0 - (got @ ref) / (gn * rn)), float(abs(gn / rn - 1.0))


def _nets(k, device=DEV):
    """a replica of the policy / value nets and their Adam states (the same seeds on every rank: replicas start identical)"""
    from uhc_b200 import nn
    if "P" in k:
        pol = nn.MCPNet(k["D"], k["hs"], k["A"], k["htype"], num_primitive=k["P"], composer_dim=k["cd"], device=device, seed=41)
    else:
        pol = nn.MLPNet(k["D"], k["hs"], k["A"], k["htype"], device=device, head_name="action_mean", seed=41)
    val = nn.MLPNet(k["D"], k["hs"], 1, k["htype"], device=device, head_name="value_head", seed=42)
    return pol, val, nn.Adam(pol.params(), LR_P, net=pol), nn.Adam(val.params(), LR_V, net=val)


class Rollout:
    """a [T][W E] lock-step rollout; shard(r) is rank r's [T][E] columns r E .. (r + 1) E - 1, whole() all of them (one trainer of W E envs)"""

    def __init__(self, k, W, seed, device=DEV):
        T, E, D, A = k["T"], k["E"], k["D"], k["A"]
        g = torch.Generator().manual_seed(seed)
        self.T, self.E, self.W, self.device = T, E, W, device
        self.states = torch.randn(T, W * E, D, generator=g).clamp(-5, 5)
        self.last = torch.randn(W * E, D, generator=g).clamp(-5, 5)
        self.actions = 0.1 * torch.randn(T, W * E, A, generator=g)
        self.rewards = torch.rand(T, W * E, generator=g)
        self.masks = (torch.rand(T, W * E, generator=g) > 0.1).float()
        self.masks[-1, ::4] = 0.0
        self.exps = (torch.rand(T, W * E, generator=g) > 0.1).float()
        self.log_std = torch.linspace(-2.5, -1.5, A).to(device)

    def _cols(self, c0, c1):
        d = lambda x: x[:, c0:c1].contiguous().to(self.device)
        T, n = self.T, c1 - c0
        return dict(states=d(self.states).reshape(T * n, -1), last=self.last[c0:c1].contiguous().to(self.device),
                    actions=d(self.actions).reshape(T * n, -1), rewards=d(self.rewards), masks=d(self.masks), exps=d(self.exps).reshape(-1), T=T, E=n)

    def shard(self, r):
        return self._cols(r * self.E, (r + 1) * self.E)

    def whole(self):
        return self._cols(0, self.W * self.E)


def _c_update(tr, sh, log_std, epochs, clip, losses, zf=None, zsync=None, comm=None, world=1):
    tr.update(sh["states"], sh["last"], sh["actions"], sh["rewards"], sh["masks"], sh["exps"], log_std, sh["T"], sh["E"], GAMMA, TAU, EPS, epochs, clip, losses,
              zfilter=zf, z_sync=zsync, comm=comm, world=world)


class Ranks:
    """W replicas, each with a uhc_ppo_update trainer that calls the loopback collective"""

    def __init__(self, k, W, Mcap=None, Ecap=None):
        from uhc_b200 import nn
        self.k, self.W = k, W
        self.group = LoopbackGroup(W)
        self.reps = [_nets(k) for _ in range(W)]
        Mcap, Ecap = Mcap or k["T"] * k["E"], Ecap or k["E"]
        self.trs = [nn.CPpoTrainer(p, v, op, ov, Mcap, Ecap, torch.device(DEV), all_reduce=self.group.fn) for p, v, op, ov in self.reps]
        D = k["D"]
        self.zf = [torch.zeros(1 + 2 * D, device=DEV, dtype=torch.float64) for _ in range(W)]
        self.zsync = [torch.zeros(1 + 2 * D, device=DEV, dtype=torch.float64) for _ in range(W)]
        self.losses = [torch.zeros(2, device=DEV) for _ in range(W)]

    def update(self, ro, epochs, clip, last=None):
        """last[r]: rank r's normalised last states (default: the rollout's)"""
        def rank(r):
            sh = ro.shard(r)
            if last is not None:
                sh["last"] = last[r]
            _c_update(self.trs[r], sh, ro.log_std, epochs, clip, self.losses[r], self.zf[r], self.zsync[r], self.group.comm(r), self.W)
        self.group.run(rank)
        torch.cuda.synchronize()

    def close(self):
        for t in self.trs:
            t.close()


def _bf16_params(net):
    return [(p.bfloat16().double() if i % 2 == 0 else p.double()).detach().clone().requires_grad_(True) for i, p in enumerate(net.params())]


def _grad_views(net):
    return [net.gflat[o:o + n].view_as(p) for (o, n), p in zip(net._offs, net.params())]


def _reference(k, ro, last_states=None):
    """fp64 of the union batch at the initial weights: (per-rank normalised advantages, per-rank returns, policy gradients, value gradients,
    surrogate loss, value loss, mean |selected advantage|).  last_states(r): rank r's normalised V(s_T) input (default: the rollout's)."""
    pol, val, _, _ = _nets(k)
    a_raw, rets = [], []
    for r in range(ro.W):
        sh = ro.shard(r)
        last = sh["last"] if last_states is None else last_states(r)
        v = val.forward_tc(sh["states"]).reshape(ro.T, ro.E).double().clone()
        vl = val.forward_tc(last).reshape(ro.E).double().clone()
        a, rt = R.gae_te(sh["rewards"].double(), sh["masks"].double(), v, GAMMA, TAU, vl)
        a_raw.append(a.reshape(-1)); rets.append(rt.reshape(-1))
    a_all = torch.cat(a_raw)
    mu, sd = a_all.mean(), a_all.std(unbiased=True)
    advs = [(a - mu) / sd for a in a_raw]
    sh = [ro.shard(r) for r in range(ro.W)]
    xs = torch.cat([s["states"] for s in sh]).bfloat16().double()
    act64, ex64 = torch.cat([s["actions"] for s in sh]).double(), torch.cat([s["exps"] for s in sh]).double()
    adv64, ret64 = torch.cat(advs), torch.cat(rets)
    pp, vp = _bf16_params(pol), _bf16_params(val)
    if "P" in k:
        n = len(pol.prims[0].params())
        mean = R.mcp([pp[j * n:(j + 1) * n] for j in range(k["P"])], pp[k["P"] * n:], xs, k["htype"], store=R.bf16_store)[0]
    else:
        mean = R.mlp(pp, xs, k["htype"], store=R.bf16_store)
    logp = R.gaussian_logp(mean, ro.log_std.double(), act64)
    lp = R.surrogate_loss(logp, logp.detach(), adv64, ex64, EPS)      # one epoch: the fixed log-probabilities come from the same weights
    lv = R.value_loss(R.mlp(vp, xs, k["htype"], store=R.bf16_store), ret64)
    return dict(adv=advs, ret=rets, gp=R.grads_of(lp, pp), gv=R.grads_of(lv, vp), lp=lp.item(), lv=lv.item(), adv_scale=float(adv64[ex64 != 0].abs().mean()))


def _check_update(tag, reps, losses, ref, p0, v0, clip):
    """one epoch of a W-rank update against the fp64 union reference: gradients bit-identical across ranks and within the single-GPU bounds of
    test_update_policy_gradients_losses_and_step; the step equals p0 + one fp64 Adam step (first-step clip) on the global gradient; the ranks'
    loss shares sum to the global loss"""
    (pol, val, _, _) = reps[0]
    for r, (p, v, _, _) in enumerate(reps[1:], 1):
        assert torch.equal(p.gflat, pol.gflat) and torch.equal(v.gflat, val.gflat), (tag, r)
        assert torch.equal(p.flat, pol.flat) and torch.equal(v.flat, val.flat), (tag, r)
    for name, net, gref in (("policy", pol, ref["gp"]), ("value", val, ref["gv"])):
        worst = [0.0, 0.0, 0.0]
        for g, rr in zip(_grad_views(net), gref):
            worst = [max(a, b) for a, b in zip(worst, _tensor_metrics(g, rr))]
        # measured over small / production / mcp / obs v3, W = 2, 3, both paths: 3.6e-3, 6.4e-6, 6.0e-4
        _check(f"{tag} {name} gradients, relative Frobenius", worst[0], 1.2e-2)
        _check(f"{tag} {name} gradients, 1 - cosine", worst[1], 3e-5)
        _check(f"{tag} {name} gradients, |norm ratio - 1|", worst[2], 3e-3)
    lsum = torch.stack(losses).double().sum(0).cpu()
    # measured 6.1e-7 and 4.3e-7 (production, W = 2 and 3)
    _check(f"{tag} sum of the ranks' surrogate losses, relative", abs(lsum[0].item() - ref["lp"]) / ref["adv_scale"], 2e-6)
    _check(f"{tag} sum of the ranks' value losses, relative", abs(lsum[1].item() - ref["lv"]) / ref["lv"], 2e-6)
    for name, net, w0, lr, mn in (("policy", pol, p0, LR_P, clip), ("value", val, v0, LR_V, None)):
        rf = w0.double().clone().requires_grad_(True)
        rf.grad = net.gflat.double().clone()
        if mn is not None:
            torch.nn.utils.clip_grad_norm_([rf], mn)
        R.adam([rf], lr).step()
        _check(f"{tag} {name} step, max |err| / lr", float((net.flat.double() - rf.detach()).abs().max()) / lr, 5e-4)     # measured 1.4e-4 (mcp)


def _active_clip(ref):
    return 0.25 * float(torch.sqrt(sum((x ** 2).sum() for x in ref["gp"])))


@pytest.fixture(scope="module", autouse=True)
def _serial_warm_up():
    """one update on the main thread before any test starts rank threads: the GEMM path's lazily initialised state is set up serially"""
    from uhc_b200 import nn
    k = dict(KINDS["small"], T=2, E=64)
    pol, val, op, ov = _nets(k)
    ro = Rollout(k, 1, seed=1)
    tr = nn.CPpoTrainer(pol, val, op, ov, 128, 64, torch.device(DEV))
    _c_update(tr, ro.whole(), ro.log_std, 1, 40.0, torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
    tr.close()


# ------------------------------------------------------------------------------------------------ the loopback collective itself
@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_loopback_all_reduce(W):
    """integer-valued floats sum exactly: every rank receives the exact sum, in place, on every one of several calls (its private buffer is
    reused); counts that differ between the ranks fail every rank and leave the buffers untouched; the group still works afterwards"""
    g = LoopbackGroup(W, timeout=30.0)
    n = 100003
    bufs = [torch.zeros(n, device=DEV) for _ in range(W)]
    base = torch.arange(n, device=DEV, dtype=torch.float32) % 977 - 300
    seen = [[] for _ in range(W)]

    def calls(r):
        out = []
        for c in range(3):
            bufs[r].copy_(base * (r + 1) + c)          # the producer runs on the rank's stream, right before the collective
            rc = g.fn(bufs[r].data_ptr(), bufs[r].data_ptr(), n, NCCL_FLOAT32, NCCL_SUM, g.comm(r).value, torch.cuda.current_stream().cuda_stream)
            out.append((rc, bufs[r].clone()))
            seen[r].append(g._priv[r].data_ptr())
        return out
    res = g.run(calls)
    for c in range(3):
        want = base * (W * (W + 1) / 2) + W * c
        for r in range(W):
            assert res[r][c][0] == 0 and torch.equal(res[r][c][1], want), (W, r, c)
    assert all(len(set(s)) == 1 for s in seen), "the private buffer was reallocated between calls of one count"
    assert g.log == [[(n, 4 * n)] * 3] * W

    def mismatch(r):
        bufs[r].fill_(float(r + 1))
        cnt = n - (r == W - 1) if W > 1 else n
        return g.fn(bufs[r].data_ptr(), bufs[r].data_ptr(), cnt, NCCL_FLOAT32, NCCL_SUM, g.comm(r).value, torch.cuda.current_stream().cuda_stream)
    rcs = g.run(mismatch)
    if W > 1:
        assert rcs == [ERR_COUNTS] * W
        assert all(torch.equal(bufs[r], torch.full((n,), float(r + 1), device=DEV)) for r in range(W))
    res = g.run(calls)
    assert all(res[r][c][0] == 0 for r in range(W) for c in range(3))


def test_loopback_refuses_and_reports():
    """a datatype other than float32 or an op other than sum is refused; an exception inside the callback returns non-zero (not ctypes' 0)"""
    x = torch.ones(8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    for dt, op in ((NCCL_FLOAT32 + 2, NCCL_SUM), (NCCL_FLOAT32, NCCL_SUM + 1)):
        g = LoopbackGroup(1, timeout=5.0)
        assert g.fn(x.data_ptr(), x.data_ptr(), 8, dt, op, g.comm(0).value, st) == ERR_REFUSED
    g = LoopbackGroup(1, timeout=5.0)
    g.all_reduce = lambda *a: 1 // 0
    assert g.fn(x.data_ptr(), x.data_ptr(), 8, NCCL_FLOAT32, NCCL_SUM, g.comm(0).value, st) == ERR_EXCEPTION
    assert "ZeroDivisionError" in g.errors[-1]


# ------------------------------------------------------------------------------------------------ a, b: one update against fp64
@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("kind", ["small", "production", "mcp"])
def test_multirank_update_matches_fp64(kind, W):
    """catches: a local row count in the value scale (norm ratio 1/W), a local selected-row count (policy norm ratio ~W), a missing statistics
    tail (local normalisation: the gradients move by ~10 %), planes joined at the wrong scale (the advantages scale by 2^k)"""
    k = KINDS[kind]
    ro = Rollout(k, W, seed=100 + W)
    ref = _reference(k, ro)
    clip = _active_clip(ref)
    rk = Ranks(k, W)
    p0, v0 = rk.reps[0][0].flat.clone(), rk.reps[0][1].flat.clone()
    rk.update(ro, 1, clip)
    _check_update(f"{kind} W={W}", rk.reps, rk.losses, ref, p0, v0, clip)
    rk.close()


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("T,E", [(8, 256), (5, 129)])
def test_multirank_advantages_and_returns(T, E, W):
    """uhc_ppo_advantages / uhc_ppo_returns of every rank against its columns' fp64 GAE and the normalisation over the union
    (catches: a local normalisation, the planes joined at a wrong scale, a wrong global row count)"""
    k = dict(KINDS["small"], T=T, E=E)
    ro = Rollout(k, W, seed=7 * T + E)
    ref = _reference(k, ro)
    rk = Ranks(k, W)
    rk.update(ro, 1, 40.0)
    M = T * E
    cudart = C.cdll.LoadLibrary("libcudart.so")
    for r, tr in enumerate(rk.trs):
        adv = tr.advantages(M).double()
        ret = torch.empty(M, device=DEV)
        cudart.cudaMemcpy(C.c_void_p(ret.data_ptr()), C.c_void_p(tr.L.uhc_ppo_returns(tr.h)), C.c_size_t(4 * M), C.c_int(3))
        # the single-GPU bounds of test_full_update_advantages_and_returns (measured here 6.2e-7, 1.9e-7)
        _check(f"advantages T={T} E={E} W={W} rank {r}", float((adv - ref["adv"][r]).abs().max()), 3e-6)
        _check(f"returns T={T} E={E} W={W} rank {r}", float((ret.double() - ref["ret"][r]).abs().max() / ref["ret"][r].abs().max()), 1e-6)
    rk.close()


# ------------------------------------------------------------------------------------------------ c: the ZFilter merge
def _obs_batch(g, n, D, shape_vec):
    """raw observations: mixed scales, column 5 with a mean 1e5 times its standard deviation, the constant shape vector in columns 640 .. 656"""
    x = torch.randn(n, D, generator=g, dtype=torch.float64) * torch.linspace(0.1, 3.0, D, dtype=torch.float64) + torch.linspace(-2.0, 2.0, D, dtype=torch.float64)
    x[:, 5] = 1000.0 + 0.01 * torch.randn(n, generator=g, dtype=torch.float64)
    x[:, 640:657] = shape_vec
    return x.float()


def _bare_agent(nets, D, world, comm=None):
    """a BatchedAgent with only what update_params and load_state_dicts read (no engine: the update runs on seeded buffers)"""
    from uhc_b200 import nn
    from uhc_b200.agent import BatchedAgent
    ag = BatchedAgent.__new__(BatchedAgent)
    ag.torch, ag.dev, ag.world, ag.obs_dim = torch, torch.device(DEV), world, D
    ag.policy, ag.value, ag.opt_p, ag.opt_v = nets
    ag.log_std = torch.linspace(-2.5, -1.5, ag.policy.dims[-1]).to(DEV)
    ag.running_state = nn.ZFilter(D, clip=5.0, device=DEV)
    ag.comm = comm
    ag.gamma, ag.tau, ag.clip_epsilon, ag.epochs, ag.grad_clip = GAMMA, TAU, EPS, 1, 40.0
    ag.update_tc, ag.c_update = True, False
    return ag


@pytest.mark.parametrize("restored", [False, True])
def test_multirank_zfilter_merge_over_three_updates(restored):
    """every rank's normaliser sees its own batches (different sizes) between updates; after each update all ranks hold the same bits, n is
    exact, mean and S match the fp64 Chan merge of every batch every rank has seen, and the constant shape-vector columns normalise to ~0.
    restored: the normaliser comes from a checkpoint (BatchedAgent.load_state_dicts) on every rank, which must count it once, not W times.
    Catches: a missing `zsync +=` (the second update counts the first one's increments again)."""
    from uhc_b200 import nn
    W, D = 3, 657
    k = dict(KINDS["small"], hs=(64,), T=4, E=32)
    rk = Ranks(k, W)
    g = torch.Generator().manual_seed(77)
    shape_vec = torch.randn(17, generator=g, dtype=torch.float64) * 0.5
    zfs = [nn.ZFilter(D, device=DEV) for _ in range(W)]
    state = P.zf_empty(D)
    if restored:
        x0 = _obs_batch(g, 500, D, shape_vec)
        s0 = P.zf_merge(P.zf_empty(D), x0.double().numpy())
        for r in range(W):
            ag = _bare_agent(rk.reps[r], D, W)
            ag.running_state = zfs[r]
            ag.load_state_dicts({"policy_dict": ag.policy.state_dict(), "value_dict": ag.value.state_dict(),
                                 "running_state": {"n": s0[0], "mean": s0[1], "std": P.zf_std(s0)}})
            rk.zsync[r] = ag._z_sync
        st = zfs[0].stats.cpu().numpy()
        state = (st[0], st[1:1 + D].copy(), st[1 + D:].copy())          # what the checkpoint restores (S through the std, as the loader does)
    for r in range(W):
        rk.zf[r] = zfs[r].stats
    worst_m = worst_s = worst_c = worst_y = 0.0
    for upd in range(3):
        for r in range(W):
            for part in range(2):
                x = _obs_batch(g, 11 + 7 * r + 13 * upd + 5 * part, D, shape_vec)
                zfs[r](x.to(DEV), update=True)
                state = P.zf_merge(state, x.double().numpy())
        ro = Rollout(k, W, seed=200 + upd)
        rk.update(ro, 1, 40.0)
        for r in range(1, W):
            assert torch.equal(zfs[r].stats, zfs[0].stats), (upd, r)
        st = zfs[0].stats.cpu().numpy()
        n, mean, S = st[0], st[1:1 + D], st[1 + D:]
        assert n == state[0], (upd, n, state[0])
        v, c = np.ones(D, dtype=bool), np.zeros(D, dtype=bool)
        v[640:657], c[640:657] = False, True
        sd = np.sqrt(state[2][v] / (state[0] - 1))
        worst_m = max(worst_m, float((np.abs(mean[v] - state[1][v]) / (sd + np.abs(state[1][v]) * 1e-9)).max()))
        worst_s = max(worst_s, float((np.abs(S[v] - state[2][v]) / state[2][v]).max()))
        worst_c = max(worst_c, float(np.abs(mean[c] - state[1][c]).max() / np.abs(shape_vec.numpy()).max()))
        xq = _obs_batch(g, 64, D, shape_vec).to(DEV)
        y = zfs[0](xq, update=False)
        assert torch.isfinite(y).all()
        worst_y = max(worst_y, float(y[:, 640:657].abs().max()))
    tag = "restored" if restored else "fresh"
    # measured (worst of both variants): 1.5e-10; 2.5e-5 (column 5, mean 1e5 std: S is a difference of sums of squares ~1e8 times larger);
    # 0 and 0 -- the constant columns' sums are exact in the 2^-30 digits at these sizes, so their S merges to 0 and they normalise to 0
    _check(f"zfilter {tag}: max |mean - fp64| / (std + 1e-9 |mean|)", worst_m, 1e-9)
    _check(f"zfilter {tag}: max |S - fp64| / S", worst_s, 1e-4)
    _check(f"zfilter {tag}: constant columns, max |mean - fp64| / |shape|", worst_c, 1e-12)
    _check(f"zfilter {tag}: constant columns, max |normalised value|", worst_y, 1e-6)
    rk.close()


# ------------------------------------------------------------------------------------------------ d: sharded equals unsharded
@pytest.mark.parametrize("kind", ["small", "mcp"])
def test_sharded_update_equals_unsharded(kind):
    """W ranks of E envs against one trainer of W E envs (the same columns), 10 epochs, two updates: the parameters agree by
    test_gpu_ppo_c's criterion between its two update paths; parameters, Adam moments and step counters are the same bits on every replica;
    each update makes two collectives per epoch of the expected sizes"""
    from uhc_b200 import nn
    W, epochs = 2, 10
    k = dict(KINDS[kind], T=4, E=128)
    rk = Ranks(k, W)
    pol1, val1, op1, ov1 = _nets(k)
    p0, v0 = pol1.flat.clone(), val1.flat.clone()
    one = nn.CPpoTrainer(pol1, val1, op1, ov1, k["T"] * k["E"] * W, k["E"] * W, torch.device(DEV))
    D = k["D"]
    pol, val = rk.reps[0][0], rk.reps[0][1]
    for upd in range(2):
        ro = Rollout(k, W, seed=300 + upd)
        _c_update(one, ro.whole(), ro.log_std, epochs, 40.0, torch.zeros(2, device=DEV))
        rk.update(ro, epochs, 40.0)
        for r in range(W):
            ms, by, calls = rk.trs[r].comm_stats()
            assert calls == 2 * epochs and by == 4 * (epochs * (pol.nflat + val.nflat) + nn.stats_tail_floats(D)), (upd, r, calls, by)
            assert [c for c, _ in rk.group.log[r]] == [val.nflat + nn.stats_tail_floats(D), pol.nflat] + [val.nflat, pol.nflat] * (epochs - 1)
            rk.group.log[r].clear()
    torch.cuda.synchronize()
    for r, (p, v, op, ov) in enumerate(rk.reps[1:], 1):
        assert torch.equal(p.flat, pol.flat) and torch.equal(v.flat, val.flat), r
        for a, b in ((op, rk.reps[0][2]), (ov, rk.reps[0][3])):
            assert torch.equal(a.mflat, b.mflat) and torch.equal(a.vflat, b.vflat) and a.step_n == b.step_n == 2 * epochs, r
    for name, w1, w2, w0, lr in (("policy", pol1.flat, pol.flat, p0, LR_P), ("value", val1.flat, val.flat, v0, LR_V)):
        d1, d2 = w1 - w0, w2 - w0
        assert d1.abs().max().item() > 0.5 * lr
        rel_mean = (d1 - d2).abs().mean().item() / d1.abs().mean().item()
        # test_gpu_ppo_c's criterion; measured 2.6e-3 and 0.10 (policy, mcp)
        _check(f"sharded {kind} {name}: mean |unsharded - sharded| / mean |update|", rel_mean, 0.02)
        _check(f"sharded {kind} {name}: max |unsharded - sharded| / (steps lr)", (d1 - d2).abs().max().item() / (2 * epochs * lr), 0.6)
    one.close()
    rk.close()


# ------------------------------------------------------------------------------------------------ e, f: the Python path and obs v3 widths
def _identity_filter_stats(D):
    """a restored normaliser of mean 0 and std 1 on every rank"""
    return {"n": 2.0, "mean": np.zeros(D), "std": np.ones(D)}


def _python_ranks(k, W, ro, epochs, clip, zbatches=None):
    """BatchedAgent.update_params on the Python path (c_update=False) of W bare agents over the loopback GradComm; zbatches[r]: observations
    rank r's normaliser takes in before the update.  Returns the agents, their logs and the normalised last states their V(s_T) read."""
    from uhc_b200.agent import RolloutBuffer
    group = LoopbackGroup(W)
    ags = []
    for r in range(W):
        ag = _bare_agent(_nets(k), k["D"], W, LoopbackGradComm(group, r))
        ag.grad_clip = clip
        ag.epochs = epochs
        ag.load_state_dicts({"policy_dict": ag.policy.state_dict(), "value_dict": ag.value.state_dict(), "running_state": _identity_filter_stats(k["D"])})
        ag.log_std.copy_(ro.log_std)
        ags.append(ag)
    bufs = []
    for r in range(W):
        sh = ro.shard(r)
        b = RolloutBuffer(ro.T, ro.E, DEV, k["A"], k["D"])
        b.states.copy_(sh["states"].reshape(ro.T, ro.E, -1)); b.actions.copy_(sh["actions"].reshape(ro.T, ro.E, -1))
        b.rewards.copy_(sh["rewards"]); b.masks.copy_(sh["masks"]); b.exps.copy_(sh["exps"].reshape(ro.T, ro.E)); b.last_obs.copy_(sh["last"])
        bufs.append(b)
        if zbatches is not None:
            ags[r].running_state(zbatches[r].to(DEV), update=True)
    last = [ags[r].running_state(bufs[r].last_obs, update=False).clone() for r in range(W)]
    logs = group.run(lambda r: ags[r].update_params(bufs[r]))
    torch.cuda.synchronize()
    return ags, logs, last


def test_python_path_matches_fp64_and_the_c_path():
    """BatchedAgent.update_params with c_update=False, W = 2: gradients and step against fp64 as the C path's test (a), the normalisers merged
    (c), and the parameters agree with uhc_ppo_update's on the same data by test_gpu_ppo_c's criterion (catches: a missing `_z_sync` update,
    a wrong tail scale or row count in the Python copy of the statistics logic)"""
    from uhc_b200 import nn
    W, k = 2, KINDS["small"]
    ro = Rollout(k, W, seed=500)
    g = torch.Generator().manual_seed(501)
    shape_vec = torch.randn(17, generator=g, dtype=torch.float64)
    zb = [_obs_batch(g, 40 + 9 * r, k["D"], shape_vec) for r in range(W)]
    clip = _active_clip(_reference(k, ro))
    ags, logs, last = _python_ranks(k, W, ro, 1, clip, zbatches=zb)
    ref = _reference(k, ro, last_states=lambda r: last[r])
    reps = [(a.policy, a.value, a.opt_p, a.opt_v) for a in ags]
    pol, val = _nets(k)[:2]
    _check_update(f"python W={W}", reps, [torch.tensor([lg["surr_loss"], lg["value_loss"]]) for lg in logs], ref, pol.flat, val.flat, clip)
    state = P.zf_merge(P.zf_merge((2.0, np.zeros(k["D"]), np.ones(k["D"])), zb[0].double().numpy()), zb[1].double().numpy())
    st = ags[0].running_state.stats.cpu().numpy()
    assert torch.equal(ags[1].running_state.stats, ags[0].running_state.stats) and st[0] == state[0]
    v = np.ones(k["D"], dtype=bool); v[640:657] = False
    _check("python zfilter: max |S - fp64| / S", float((np.abs(st[1 + k["D"]:][v] - state[2][v]) / state[2][v]).max()), 1e-4)      # measured 1.6e-10
    assert logs[0]["allreduce_calls"] == 2 and logs[0]["allreduce_bytes"] == 4 * (val.nflat + val.grad_tail + pol.nflat)
    # the C path on the same data and the same starting normaliser
    rk = Ranks(k, W)
    for r in range(W):
        zf = nn.ZFilter(k["D"], device=DEV)
        zf.load(**_identity_filter_stats(k["D"]))
        rk.zsync[r] = nn.zfilter_to_sums(zf.stats, k["D"]).clone()
        zf(zb[r].to(DEV), update=True)
        rk.zf[r] = zf.stats
    rk.update(ro, 1, clip, last=last)
    assert torch.equal(rk.zf[0][0], ags[0].running_state.stats[0])
    _check("python vs C zfilter, max |mean diff|", float((rk.zf[0][1:1 + k["D"]] - ags[0].running_state.stats[1:1 + k["D"]]).abs().max()), 1e-9)   # measured 0
    w0 = pol.flat
    for name, a, b, w in (("policy", ags[0].policy.flat, rk.reps[0][0].flat, w0), ("value", ags[0].value.flat, rk.reps[0][1].flat, val.flat)):
        d1, d2 = a - w, b - w
        _check(f"python vs C {name}: mean |diff| / mean |update|", (d1 - d2).abs().mean().item() / d1.abs().mean().item(), 3e-7)     # measured 3.4e-8
    rk.close()


@pytest.mark.parametrize("path", ["c", "python"])
@pytest.mark.parametrize("kind", ["v3", "v3s"])
def test_obs_v3_widths(kind, path):
    """D = 6400 / 3285 (obs v3 without / with the shape vector): the statistics tail needs 5 (5 + 2 D) floats, more than the fixed 8192 the
    gradient tensors used to have; with the tail sized from the input width both paths match fp64 as for D = 657"""
    W, k = 2, KINDS[kind]
    ro = Rollout(k, W, seed=600 + k["D"])
    ref = _reference(k, ro)
    clip = _active_clip(ref)
    pol, val = _nets(k)[:2]
    if path == "c":
        rk = Ranks(k, W)
        rk.update(ro, 1, clip)
        _check_update(f"{kind} C", rk.reps, rk.losses, ref, pol.flat, val.flat, clip)
        rk.close()
    else:
        ags, logs, last = _python_ranks(k, W, ro, 1, clip)
        ref = _reference(k, ro, last_states=lambda r: last[r])
        _check_update(f"{kind} python", [(a.policy, a.value, a.opt_p, a.opt_v) for a in ags],
                      [torch.tensor([lg["surr_loss"], lg["value_loss"]]) for lg in logs], ref, pol.flat, val.flat, clip)


# ------------------------------------------------------------------------------------------------ g: refusals
def test_update_policy_refuses_world_above_one():
    """uhc_ppo_update_policy would divide the policy gradient by this rank's selected-row count (W times the global mean after the sum)"""
    from uhc_b200 import nn
    k = dict(KINDS["small"], T=2, E=64)
    pol, val, op, ov = _nets(k)
    tr = nn.CPpoTrainer(pol, val, op, ov, 128, 64, torch.device(DEV))
    sh = Rollout(k, 1, seed=3).whole()
    p0, v0 = pol.flat.clone(), val.flat.clone()
    cfg = nn.UhcPpoCfg(0.0, 0.0, EPS, 40.0, 1, 1)
    sp, sv, done = C.c_int(0), C.c_int(0), C.c_int(0)
    z = torch.zeros(128, device=DEV)
    rc = tr.L.uhc_ppo_update_policy(tr.h, nn._p(sh["states"]), nn._p(sh["actions"]), nn._p(z), nn._p(z), nn._p(sh["exps"]), nn._p(torch.full((105,), -2.3, device=DEV)),
                                    C.c_long(128), C.byref(cfg), C.byref(sp), C.byref(sv), C.byref(done), C.c_void_p(1), C.c_int(2), nn._p(torch.zeros(2, device=DEV)), nn._stream(z))
    torch.cuda.synchronize()
    assert rc == -2 and b"world > 1" in tr.L.uhc_last_error()
    assert torch.equal(pol.flat, p0) and torch.equal(val.flat, v0) and sp.value == 0 and sv.value == 0
    tr.close()


def test_fp32_update_refuses_world_above_one():
    """the fp32 update path has no gradient all-reduce: its replicas would drift apart silently"""
    from uhc_b200.agent import BatchedAgent
    with pytest.raises(ValueError, match="single-GPU"):
        BatchedAgent(8, [], world=2, update_tc=False)


def test_failed_collective_fails_the_update_and_the_next_one_succeeds():
    from uhc_b200 import nn
    W = 2
    k = dict(KINDS["small"], T=2, E=64)
    rk = Ranks(k, W)
    calls = []

    def failing(send, recv, count, dtype, op, comm, stream):
        calls.append(count)
        return 5
    bad = nn.ALL_REDUCE_FN(failing)
    tr, (pol, val, op, ov) = rk.trs[0], rk.reps[0]
    assert tr.L.uhc_ppo_trainer_set_all_reduce(tr.h, bad) == 0
    ro = Rollout(k, W, seed=9)
    p0, v0 = pol.flat.clone(), val.flat.clone()
    with pytest.raises(RuntimeError, match="all-reduce .*failed with code 5"):
        _c_update(tr, ro.shard(0), ro.log_std, 1, 40.0, rk.losses[0], rk.zf[0], rk.zsync[0], rk.group.comm(0), W)
    torch.cuda.synchronize()
    assert calls == [val.nflat + nn.stats_tail_floats(k["D"])]
    assert torch.equal(pol.flat, p0) and torch.equal(val.flat, v0) and op.step_n == 0 and ov.step_n == 0
    assert tr.L.uhc_ppo_trainer_set_all_reduce(tr.h, rk.group.fn) == 0
    rk.update(ro, 1, 40.0)
    assert op.step_n == 1 and not torch.equal(pol.flat, p0) and torch.equal(pol.flat, rk.reps[1][0].flat)
    assert rk.trs[0].comm_stats()[2] == 2
    rk.close()


# ------------------------------------------------------------------------------------------------ h: real NCCL across GPUs
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _nccl_worker(rank, world, port, kind, epochs, clip, q):
    import torch.distributed as dist
    from uhc_b200 import nn
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        dev = torch.device("cuda", rank)
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", rank=rank, world_size=world)
        comm = nn.make_nccl_comm(rank, world, dev)
        k = KINDS[kind]
        ro = Rollout(k, world, seed=700, device=dev)
        pol, val, op, ov = _nets(k, device=dev)
        tr = nn.CPpoTrainer(pol, val, op, ov, k["T"] * k["E"], k["E"], dev)
        zf = torch.zeros(1 + 2 * k["D"], device=dev, dtype=torch.float64)
        _c_update(tr, ro.shard(rank), ro.log_std, epochs, clip, torch.zeros(2, device=dev), zf, torch.zeros_like(zf), comm, world)
        torch.cuda.synchronize()
        q.put((rank, pol.gflat.cpu(), val.gflat.cpu(), pol.flat.cpu(), val.flat.cpu(), None))
        tr.close()
        dist.destroy_process_group()
    except BaseException as e:
        q.put((rank, None, None, None, None, repr(e)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="real NCCL needs two or more visible GPUs")
@pytest.mark.parametrize("epochs", [1, 10])
def test_nccl_matches_loopback(epochs):
    """min(4, GPUs) processes on ncclAllReduce (nn.make_nccl_comm) against the loopback on the same data: one epoch (a) and ten (d)"""
    import torch.multiprocessing as mp
    W, kind = min(4, torch.cuda.device_count()), "small"
    k = KINDS[kind]
    ro = Rollout(k, W, seed=700)
    clip = _active_clip(_reference(k, ro))
    rk = Ranks(k, W)
    rk.update(ro, epochs, clip)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_nccl_worker, args=(r, W, port, kind, epochs, clip, q)) for r in range(W)]
    for p in ps:
        p.start()
    try:
        res = sorted((q.get(timeout=600) for _ in ps), key=lambda x: x[0])
    finally:
        for p in ps:
            p.join(60)
        for p in ps:
            if p.is_alive():
                p.terminate()
                p.join(10)
    assert all(x[5] is None for x in res), [x[5] for x in res]
    pol, val = rk.reps[0][0], rk.reps[0][1]
    p0, v0 = _nets(k)[:2]
    for r, gp, gv, fp, fv, _ in res:
        if epochs == 1:
            for name, g, ref_net in (("policy", gp, pol), ("value", gv, val)):
                m = _tensor_metrics(g, ref_net.gflat.cpu())
                _check(f"nccl W={W} rank {r} {name} gradients vs loopback, relative Frobenius", m[0], 1.2e-2)
                _check(f"nccl W={W} rank {r} {name} gradients vs loopback, 1 - cosine", m[1], 3e-5)
        for name, f, ref_net, w0, lr in (("policy", fp, pol, p0.flat, LR_P), ("value", fv, val, v0.flat, LR_V)):
            d1, d2 = ref_net.flat.cpu() - w0.cpu(), f - w0.cpu()
            _check(f"nccl W={W} rank {r} {name} epochs={epochs}: mean |diff| / mean |update|", (d1 - d2).abs().mean().item() / d1.abs().mean().item(), 0.02)
    rk.close()
