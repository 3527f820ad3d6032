"""Policy / value networks, Gaussian head, ZFilter, GAE and the PPO update on the hand-written kernels (include/uhc_nn.h).

PyTorch tensors hold the parameters (so the reference's pickle checkpoint format -- a state_dict with the keys
net.affine_layers.{i}.{weight,bias}, action_mean.*, action_log_std, value_head.* -- round-trips unchanged,
uhc/agents/agent_copycat.py:190-201); every arithmetic op below is a kernel of libuhc_b200.so, not torch.
"""
import ctypes as C
import math

import numpy as np

from .engine import _chk as _check, load_library as _lib

ACT = {"none": 0, "gelu": 1, "tanh": 2, "relu": 3, "sigmoid": 4}


def _chk(rc):
    _check(rc, "uhc_nn")


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def _stream(t):
    import torch
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def stats_tail_floats(in_dim):
    """floats after a net's gradients in its flat gradient tensor: a world > 1 update carries its global statistics there through the value
    gradient's all-reduce, as split_double's 5 digit planes of [advantage sum, sum of squares, rows, selected rows, the ZFilter increment
    (n, sum[D], sum of squares[D])], 5 (5 + 2 D) floats for an input width D (include/uhc_ppo.h UhcNetDesc.gtail)"""
    return SPLIT_CHUNKS * (4 + 1 + 2 * in_dim)


def linear_forward(x, W, b, act="none", save_z=False):
    import torch
    M, K = x.shape
    N = W.shape[0]
    y = torch.empty(M, N, device=x.device, dtype=torch.float32)
    z = torch.empty_like(y) if save_z else None
    _chk(_lib().uhc_linear_forward(_p(x), _p(W), _p(b), _p(y), _p(z), M, N, K, ACT[act], _stream(x)))
    return (y, z) if save_z else y


class ParamList(list):
    """params() of an MLPNet: a plain list that remembers its net (so an optimiser built from it can work on the flat tensors)"""
    net = None


class MLPNet:
    """MLP trunk + linear head (khrylib/models/mlp.py:5-27 with PolicyGaussian.action_mean or Value.value_head)."""

    @staticmethod
    def flat_layout(dims):
        """offsets (start, count) of W[0], b[0], W[1], ... in the flat tensor (every tensor starts on a 256-byte boundary) and the total length"""
        offs, o = [], 0
        for i in range(len(dims) - 1):
            nW, nb = dims[i + 1] * dims[i], dims[i + 1]
            offs.append((o, nW)); o += (nW + 63) // 64 * 64
            offs.append((o, nb)); o += (nb + 63) // 64 * 64
        return offs, o

    def __init__(self, in_dim, hsize, out_dim, htype="gelu", device="cuda", head_name="action_mean", seed=None, storage=None, head_act="none",
                 head_scale=(0.1, 0.0), generator=None):
        """storage = (flat, gfull, base): this net's parameters / gradients are the slice [base, base + nflat) of a shared flat tensor (PolicyMCP: all
        primitives and the composer live in one tensor -> one all-reduce, one Adam launch); head_act: activation after the output layer (the MCP
        composer is a plain MLP whose last layer is activated too, mlp.py:24-27); head_scale: (weight, bias) factors of the output layer's init."""
        import torch
        self.torch, self.dims, self.htype, self.head_name = torch, [in_dim] + list(hsize) + [out_dim], htype, head_name
        self.head_act = head_act
        g = generator if generator is not None else (torch.Generator().manual_seed(seed) if seed is not None else None)
        # ONE flat fp32 tensor holds every parameter (each tensor starts on a 256-byte boundary), W[i] / b[i] are views of it; the
        # gradients live in an identically laid out flat tensor (`gflat`) with a small tail for the scalar statistics that ride the
        # gradient all-reduce (SURVEY.md section 8e) -- so Adam is one launch per net and the collective needs no flatten / copy.
        offs, o = self.flat_layout(self.dims)
        self._offs, self.nflat = offs, o
        self.grad_tail = stats_tail_floats(in_dim)
        self._storage = storage
        if storage is None:
            self.flat = torch.zeros(o, device=device, dtype=torch.float32)
            self._gfull = None
        else:
            sflat, sgfull, base = storage
            self.flat, self._gfull, self._base = sflat[base:base + o], sgfull[base:base + o], base
        self.W, self.b = [], []
        for i in range(len(self.dims) - 1):  # nn.Linear default init: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias
            k = 1.0 / math.sqrt(self.dims[i])
            # explicit dtype: the reference's scripts set torch.set_default_dtype(float64) (train_uhc.py:80-81); the seeded stream must not depend on it
            w = (torch.rand(self.dims[i + 1], self.dims[i], generator=g, dtype=torch.float32) * 2 - 1) * k
            bb = (torch.rand(self.dims[i + 1], generator=g, dtype=torch.float32) * 2 - 1) * k
            if i == len(self.dims) - 2 and head_scale is not None:  # policy_gaussian.py:20-21 / critic.py:12-13 / policy_mcp.py:20-22
                w, bb = w * head_scale[0], bb * head_scale[1]
            (ow, nw), (ob, nb) = offs[2 * i], offs[2 * i + 1]
            W, B = self.flat[ow:ow + nw].view(self.dims[i + 1], self.dims[i]), self.flat[ob:ob + nb]
            W.copy_(w.float()); B.copy_(bb.float())
            self.W.append(W)
            self.b.append(B)
        self.device = device
        self._bf16 = None
        self.opt = None

    # ---- state_dict in the reference's key layout
    def state_dict(self):
        sd = {}
        n = len(self.W)
        for i in range(n - 1):
            sd[f"net.affine_layers.{i}.weight"], sd[f"net.affine_layers.{i}.bias"] = self.W[i].detach().cpu(), self.b[i].detach().cpu()
        sd[f"{self.head_name}.weight"], sd[f"{self.head_name}.bias"] = self.W[-1].detach().cpu(), self.b[-1].detach().cpu()
        return sd

    def load_state_dict(self, sd):
        t = self.torch
        n = len(self.W)
        for i in range(n - 1):
            self.W[i].copy_(t.as_tensor(np.asarray(sd[f"net.affine_layers.{i}.weight"]), dtype=t.float32))
            self.b[i].copy_(t.as_tensor(np.asarray(sd[f"net.affine_layers.{i}.bias"]), dtype=t.float32))
        self.W[-1].copy_(t.as_tensor(np.asarray(sd[f"{self.head_name}.weight"]), dtype=t.float32))
        self.b[-1].copy_(t.as_tensor(np.asarray(sd[f"{self.head_name}.bias"]), dtype=t.float32))
        self._bf16 = None

    def params(self):
        out = ParamList(p for wb in zip(self.W, self.b) for p in wb)
        out.net = self
        return out

    @property
    def gfull(self):
        """flat gradients + tail, allocated on first use (a net living in shared storage sees its slice of the owner's gradient tensor, no tail)"""
        if self._gfull is None:
            self._gfull = self.torch.zeros(self.nflat + self.grad_tail, device=self.flat.device, dtype=self.torch.float32)
        return self._gfull

    @property
    def gflat(self):
        return self.gfull[:self.nflat]

    def ensure_grad_tail(self, n):
        """grow the tail behind the gradients to at least n floats (a world > 1 update's extra payload rides there after the statistics).
        Returns True when it grew: the gradient tensor is then a new one, and a descriptor holding its address (CPpoTrainer) must be rebuilt."""
        if n <= self.grad_tail:
            return False
        assert self._storage is None, "a net in shared storage has no tail of its own"
        g = self.torch.zeros(self.nflat + n, device=self.flat.device, dtype=self.torch.float32)
        if self._gfull is not None:
            g[:self._gfull.numel()].copy_(self._gfull)
        self._gfull, self.grad_tail = g, n
        return True

    def _act_of(self, i):
        return self.htype if i < len(self.W) - 1 else self.head_act

    def grad_views(self):
        """gradient tensors (views of gflat) in params() order"""
        g, out = self.gflat, []
        for (o, n), p in zip(self._offs, self.params()):
            out.append(g[o:o + n].view_as(p))
        return out

    # ---- fp32 path (training; exact-gelu, SIMT GEMM)
    def forward(self, x, save=False):
        h, saved = x, [x]
        n = len(self.W)
        zs = []
        for i in range(n):
            act = self._act_of(i)
            if save and i < n - 1:
                h, z = linear_forward(h, self.W[i], self.b[i], act, save_z=True)
                zs.append(z)
                saved.append(h)
            else:
                h = linear_forward(h, self.W[i], self.b[i], act)
        return (h, (saved, zs)) if save else h

    def backward(self, dy, ctx):
        """dy: [M, out] gradient wrt the head output; returns grads in params() order."""
        t = self.torch
        saved, zs = ctx
        n = len(self.W)
        grads = [None] * (2 * n)
        dz = dy.contiguous()
        L = _lib()
        for i in range(n - 1, -1, -1):
            x = saved[i]
            M, K = x.shape
            N = self.W[i].shape[0]
            dW, db = t.empty_like(self.W[i]), t.empty_like(self.b[i])
            dx = t.empty(M, K, device=x.device, dtype=t.float32) if i > 0 else None
            _chk(L.uhc_linear_backward(_p(x), _p(self.W[i]), _p(dz), _p(dx), _p(dW), _p(db), M, N, K, _stream(x)))
            grads[2 * i], grads[2 * i + 1] = dW, db
            if i > 0:
                _chk(L.uhc_act_backward(_p(dx), _p(zs[i - 1]), _p(dx), C.c_long(dx.numel()), ACT[self.htype], _stream(x)))
                dz = dx
        return grads

    # ---- tensor-core path (rollout): bf16 operands, fp32 accumulate, fused bias + activation
    def _prep_bf16(self):
        """bf16 K-padded copies of the weights for the tensor-core kernels; the tensors keep their addresses across refreshes (the
        rollout's CUDA graph holds the pointers)."""
        t = self.torch
        store = getattr(self, "_bf16_store", None)
        if store is None:
            store = [t.zeros(w.shape[0], (w.shape[1] + 63) // 64 * 64, device=w.device, dtype=t.bfloat16) for w in self.W]
            self._bf16_store = store
        for w, wb in zip(self.W, store):
            N, K = w.shape
            _chk(_lib().uhc_f32_to_bf16_padded(_p(w), _p(wb), N, K, wb.shape[1], _stream(w)))
        self._bf16 = store

    def invalidate_bf16(self):
        self._bf16 = None

    def forward_tc(self, x):
        t = self.torch
        if self._bf16 is None:
            self._prep_bf16()
        M, K = x.shape
        Kp = self._bf16[0].shape[1]
        key = (M, x.device)
        if getattr(self, "_act_key", None) != key:  # activation buffers, zero padded once
            self._acts = [t.zeros(M, w.shape[1], device=x.device, dtype=t.bfloat16) for w in self._bf16]
            self._out = t.empty(M, self.dims[-1], device=x.device, dtype=t.float32)
            self._act_key = key
        L = _lib()
        _chk(L.uhc_f32_to_bf16_padded(_p(x), _p(self._acts[0]), M, K, Kp, _stream(x)))
        n = len(self.W)
        for i in range(n):
            last = i == n - 1
            ybf = None if last else self._acts[i + 1]
            _chk(L.uhc_linear_forward_tc(_p(self._acts[i]), _p(self._bf16[i]), _p(self.b[i]), _p(ybf), _p(self._out if last else None), M,
                                         self.W[i].shape[0], self._bf16[i].shape[1], 0 if last else ybf.shape[1],
                                         ACT[self._act_of(i)], _stream(x)))
        return self._out


class UhcMlp(C.Structure):
    """include/uhc_rollout.h UhcMlp"""
    _fields_ = [("nlayers", C.c_int), ("act", C.c_int), ("dims", C.c_int * 10), ("kp", C.c_int * 8), ("W_bf16", C.c_void_p * 8), ("bias", C.c_void_p * 8)]


def mlp_struct(net):
    """UhcMlp view of an MLPNet's current bf16 weights (rebuilt after every optimiser step: _prep_bf16 allocates new tensors)."""
    if net._bf16 is None:
        net._prep_bf16()
    m = UhcMlp()
    m.nlayers, m.act = len(net.W), ACT[net.htype]
    for i, d in enumerate(net.dims):
        m.dims[i] = d
    for i, (wb, b) in enumerate(zip(net._bf16, net.b)):
        m.kp[i] = wb.shape[1]
        m.W_bf16[i] = wb.data_ptr()
        m.bias[i] = b.data_ptr()
    m._keep = (list(net._bf16), list(net.b))
    return m


class UhcMcp(C.Structure):
    """include/uhc_rollout.h UhcMcp"""
    _fields_ = [("nprim", C.c_int), ("reserved", C.c_int), ("prim", UhcMlp * 8), ("composer", UhcMlp)]


class MCPNet:
    """PolicyMCP (uhc/models/policy_mcp.py:9-37, actor_type "mcp"): num_primitive MLPs state -> policy_hsize -> action (head weight x 0.1, bias 0) and a
    composer MLP state -> composer_dim -> num_primitive whose every layer is activated, then a softmax; action_mean = sum_k w_k prim_k(x).
    All parameters live in ONE flat tensor (and the gradients in one), the sub-nets are views: Adam and the gradient all-reduce see a single net."""
    def __init__(self, in_dim, hsize, out_dim, htype="relu", num_primitive=8, composer_dim=(300, 200), device="cuda", seed=None):
        import torch
        self.torch, self.htype, self.num_primitive, self.head_name = torch, htype, num_primitive, "mcp"
        self.dims = [in_dim] + list(hsize) + [out_dim]
        pd, cd = [in_dim] + list(hsize) + [out_dim], [in_dim] + list(composer_dim) + [num_primitive]
        n_p, n_c = MLPNet.flat_layout(pd)[1], MLPNet.flat_layout(cd)[1]
        self.nflat, self.grad_tail = num_primitive * n_p + n_c, stats_tail_floats(in_dim)
        self.flat = torch.zeros(self.nflat, device=device, dtype=torch.float32)
        self.gfull = torch.zeros(self.nflat + self.grad_tail, device=device, dtype=torch.float32)
        g = torch.Generator().manual_seed(seed) if seed is not None else None
        self.prims = [MLPNet(in_dim, hsize, out_dim, htype, device=device, storage=(self.flat, self.gfull, k * n_p), generator=g) for k in range(num_primitive)]
        self.composer = MLPNet(in_dim, composer_dim, num_primitive, htype, device=device, storage=(self.flat, self.gfull, num_primitive * n_p), head_act=htype,
                               head_scale=None, generator=g)
        self.nets = self.prims + [self.composer]
        self._offs = [(n._base + o, cnt) for n in self.nets for (o, cnt) in n._offs]      # params() order, offsets into the shared flat tensor
        self.W = [w for n in self.nets for w in n.W]           # every weight matrix (parameter counts, bf16 refresh checks)
        self.b = [b for n in self.nets for b in n.b]
        self.device, self.opt = device, None

    @property
    def gflat(self):
        return self.gfull[:self.nflat]

    @property
    def _bf16(self):
        return None if any(n._bf16 is None for n in self.nets) else [w for n in self.nets for w in n._bf16]

    @_bf16.setter
    def _bf16(self, v):
        for n in self.nets:
            n._bf16 = n._bf16_store if v is not None else None

    def _prep_bf16(self):
        for n in self.nets:
            n._prep_bf16()

    def invalidate_bf16(self):
        for n in self.nets:
            n.invalidate_bf16()

    def params(self):
        out = ParamList(p for n in self.nets for wb in zip(n.W, n.b) for p in wb)
        out.net = self
        return out

    # ---- state_dict in the reference's key layout: nets.{k}.0.affine_layers.{i}.* (MLP), nets.{k}.1.* (action_mean), composer.0.affine_layers.{i}.*
    def state_dict(self):
        sd = {}
        for k, n in enumerate(self.prims):
            for i in range(len(n.W) - 1):
                sd[f"nets.{k}.0.affine_layers.{i}.weight"], sd[f"nets.{k}.0.affine_layers.{i}.bias"] = n.W[i].detach().cpu(), n.b[i].detach().cpu()
            sd[f"nets.{k}.1.weight"], sd[f"nets.{k}.1.bias"] = n.W[-1].detach().cpu(), n.b[-1].detach().cpu()
        for i in range(len(self.composer.W)):
            sd[f"composer.0.affine_layers.{i}.weight"], sd[f"composer.0.affine_layers.{i}.bias"] = self.composer.W[i].detach().cpu(), self.composer.b[i].detach().cpu()
        return sd

    def load_state_dict(self, sd):
        t = self.torch
        cp = lambda dst, src: dst.copy_(t.as_tensor(np.asarray(src), dtype=t.float32))
        for k, n in enumerate(self.prims):
            for i in range(len(n.W) - 1):
                cp(n.W[i], sd[f"nets.{k}.0.affine_layers.{i}.weight"]); cp(n.b[i], sd[f"nets.{k}.0.affine_layers.{i}.bias"])
            cp(n.W[-1], sd[f"nets.{k}.1.weight"]); cp(n.b[-1], sd[f"nets.{k}.1.bias"])
        for i in range(len(self.composer.W)):
            cp(self.composer.W[i], sd[f"composer.0.affine_layers.{i}.weight"]); cp(self.composer.b[i], sd[f"composer.0.affine_layers.{i}.bias"])
        self.invalidate_bf16()

    def _mix(self, xall, c):
        t = self.torch
        M, A, P = c.shape[0], self.dims[-1], self.num_primitive
        mean = t.empty(M, A, device=c.device, dtype=t.float32)
        _chk(_lib().uhc_mcp_combine(_p(xall), _p(c), None, _p(mean), M, A, P, _stream(c)))
        return mean

    def forward(self, x):
        """fp32 SIMT GEMMs (the parity path against the reference's fp64 torch)"""
        xall = self.torch.stack([n.forward(x) for n in self.prims]).contiguous()
        return self._mix(xall, self.composer.forward(x).contiguous())

    def forward_tc(self, x):
        """tensor-core path (what uhc_rollout_mcp / uhc_policy_forward_mcp run)"""
        xall = self.torch.stack([n.forward_tc(x).clone() for n in self.prims]).contiguous()
        return self._mix(xall, self.composer.forward_tc(x).contiguous())


def mcp_struct(net):
    """UhcMcp view of an MCPNet's current bf16 weights"""
    m = UhcMcp()
    m.nprim = net.num_primitive
    keep = []
    for k, n in enumerate(net.prims):
        s_ = mlp_struct(n); keep.append(s_)
        m.prim[k] = s_
    sc = mlp_struct(net.composer); keep.append(sc)
    m.composer = sc
    m._keep = keep
    return m


def _buf(cache, key, shape, dtype, device, zero=True):
    import torch
    t = cache.get(key)
    if t is None or tuple(t.shape) != tuple(shape):
        t = (torch.zeros if zero else torch.empty)(*shape, device=device, dtype=dtype)
        cache[key] = t
    return t


def _pad64(n):
    return (n + 63) // 64 * 64


class TCTrainer:
    """Tensor-core (wgmma, bf16 operands / fp32 accumulate) forward + backward of an MLPNet for the PPO update:
    forward stores bf16 activations and fp32 pre-activations; dX = dZ W and dW = dZ^T X run on the same TN GEMM kernel using
    transposed bf16 copies; dz = dh * act'(z), its transpose and the bias gradient come from one fused kernel."""

    def __init__(self, net):
        self.net, self.cache = net, {}

    def prepare_input(self, x):
        import torch
        M, K = x.shape
        Kp, Mp = _pad64(K), _pad64(M)
        xb = _buf(self.cache, "xb", (M, Kp), torch.bfloat16, x.device)
        _chk(_lib().uhc_f32_to_bf16_padded(_p(x), _p(xb), M, K, Kp, _stream(x)))
        xT = _buf(self.cache, "xT", (K, Mp), torch.bfloat16, x.device)
        _chk(_lib().uhc_transpose_bf16(_p(xb), _p(xT), M, K, Kp, Mp, _stream(x)))
        return xb, xT

    def forward(self, xb):
        import torch
        net, L = self.net, _lib()
        if net._bf16 is None:
            net._prep_bf16()
        M = xb.shape[0]
        acts, zs = [xb], []
        n = len(net.W)
        out = _buf(self.cache, "out", (M, net.dims[-1]), torch.float32, xb.device, zero=False)
        for i in range(n):
            last = i == n - 1
            N = net.W[i].shape[0]
            ybf = None if last else _buf(self.cache, f"a{i}", (M, _pad64(N)), torch.bfloat16, xb.device)
            z = None if last else _buf(self.cache, f"z{i}", (M, N), torch.float32, xb.device, zero=False)
            if not last and L.uhc_tc_tma_store_enabled():      # the epilogue also stores the transposed activation the dW GEMM of the backward pass reads
                yT = _buf(self.cache, f"hT{i + 1}", (N, _pad64(M)), torch.bfloat16, xb.device)
                _chk(L.uhc_linear_forward_tc_train_t(_p(acts[i]), _p(net._bf16[i]), _p(net.b[i]), _p(ybf), _p(yT), yT.shape[1], _p(z), M, N,
                                                     net._bf16[i].shape[1], ybf.shape[1], ACT[net.htype], _stream(xb)))
                self.cache[f"hT_fresh{i + 1}"] = True
            else:
                _chk(L.uhc_linear_forward_tc_train(_p(acts[i]), _p(net._bf16[i]), _p(net.b[i]), _p(ybf), _p(out if last else None), _p(z), M, N,
                                                   net._bf16[i].shape[1], 0 if last else ybf.shape[1], ACT["none" if last else net.htype], _stream(xb)))
                self.cache[f"hT_fresh{i + 1}"] = False
            if not last:
                acts.append(ybf)
                zs.append(z)
        return out, (acts, zs)

    def backward(self, dy, ctx, xT):
        import torch
        net, L = self.net, _lib()
        acts, zs = ctx
        n = len(net.W)
        M = dy.shape[0]
        Mp = _pad64(M)
        dev = dy.device
        grads = net.grad_views()     # dW / db are written straight into the flat gradient tensor the optimiser and the all-reduce use
        dh = dy.contiguous()
        fuse = bool(L.uhc_tc_tma_store_enabled()) and net.htype != "none"
        have_dz = False
        for i in range(n - 1, -1, -1):
            N, K = net.W[i].shape
            Np = _pad64(N)
            db = grads[2 * i + 1]
            if have_dz:                      # produced by the layer above's fused dX + activation-backward GEMM
                dz, dzT = dz_next, dzT_next
            else:
                dz = _buf(self.cache, f"dz{i}", (M, Np), torch.bfloat16, dev)
                dzT = _buf(self.cache, f"dzT{i}", (N, Mp), torch.bfloat16, dev)
                _chk(L.uhc_dact_bf16(_p(dh), _p(zs[i] if i < n - 1 else None), _p(dz), _p(dzT), _p(db), M, N, Np, Mp, ACT[net.htype], _stream(dy)))
            have_dz = False
            if i == 0:
                hT = xT
            else:
                hT = _buf(self.cache, f"hT{i}", (K, Mp), torch.bfloat16, dev)
                if not self.cache.get(f"hT_fresh{i}"):
                    _chk(L.uhc_transpose_bf16(_p(acts[i]), _p(hT), M, K, acts[i].shape[1], Mp, _stream(dy)))
            dW = grads[2 * i]
            _chk(L.uhc_linear_forward_tc(_p(dzT), _p(hT), None, None, _p(dW), N, K, Mp, 0, 0, _stream(dy)))      # dW = dz^T h
            if i > 0:
                WT = _buf(self.cache, f"WT{i}", (K, Np), torch.bfloat16, dev)
                _chk(L.uhc_transpose_bf16(_p(net._bf16[i]), _p(WT), N, K, net._bf16[i].shape[1], Np, _stream(dy)))
                if fuse and K % 4 == 0:
                    dz_next = _buf(self.cache, f"dz{i - 1}", (M, _pad64(K)), torch.bfloat16, dev)
                    dzT_next = _buf(self.cache, f"dzT{i - 1}", (K, Mp), torch.bfloat16, dev)
                    _chk(L.uhc_linear_dx_dact_tc(_p(dz), _p(WT), _p(zs[i - 1]), _p(dz_next), _p(dzT_next), _p(grads[2 * i - 1]), M, K, Np, _pad64(K), Mp,
                                                 ACT[net.htype], _stream(dy)))
                    have_dz = True
                else:
                    dhp = _buf(self.cache, f"dh{i}", (M, K), torch.float32, dev, zero=False)
                    _chk(L.uhc_linear_forward_tc(_p(dz), _p(WT), None, None, _p(dhp), M, K, Np, 0, 0, _stream(dy)))    # dh_prev = dz W
                    dh = dhp
        return net.gflat


class Adam:
    """torch.optim.Adam semantics (lr, betas (0.9, 0.999), eps 1e-8, no weight decay) on the fused kernel."""

    def __init__(self, params, lr, net=None):
        """net: the MLPNet whose flat parameter tensor `params` are views of -- then step() on the net's flat gradient tensor is ONE
        fused launch (plus one norm reduction when clipping) instead of one per tensor."""
        import torch
        net = net if net is not None else getattr(params, "net", None)
        self.params, self.lr, self.step_n, self.net = params, lr, 0, net
        if net is not None:
            self.mflat, self.vflat = torch.zeros_like(net.flat), torch.zeros_like(net.flat)
            self.m = [self.mflat[o:o + n].view_as(p) for (o, n), p in zip(net._offs, params)]
            self.v = [self.vflat[o:o + n].view_as(p) for (o, n), p in zip(net._offs, params)]
        else:
            self.m = [torch.zeros_like(p) for p in params]
            self.v = [torch.zeros_like(p) for p in params]
        self.sq = torch.zeros(1, device=params[0].device, dtype=torch.float64)

    def step(self, grads, max_norm=None):
        L = _lib()
        self.step_n += 1
        if self.net is not None and not isinstance(grads, (list, tuple)):     # flat gradient tensor (padding elements are zero and stay zero)
            g, p = grads, self.net.flat
            assert g.numel() == p.numel() and g.is_contiguous()
            sq = None
            if max_norm is not None:
                self.sq.zero_()
                _chk(L.uhc_sqsum(_p(g), C.c_long(g.numel()), _p(self.sq), _stream(g)))
                sq = self.sq
            _chk(L.uhc_adam_step(_p(p), _p(g), _p(self.mflat), _p(self.vflat), C.c_long(p.numel()), C.c_float(self.lr), C.c_float(0.9), C.c_float(0.999),
                                 C.c_float(1e-8), self.step_n, _p(sq), C.c_float(max_norm or 0.0), _stream(p)))
            return
        sq = None
        if max_norm is not None:
            self.sq.zero_()
            for g in grads:
                _chk(L.uhc_sqsum(_p(g), C.c_long(g.numel()), _p(self.sq), _stream(g)))
            sq = self.sq
        for p, g, m, v in zip(self.params, grads, self.m, self.v):
            _chk(L.uhc_adam_step(_p(p), _p(g), _p(m), _p(v), C.c_long(p.numel()), C.c_float(self.lr), C.c_float(0.9), C.c_float(0.999),
                                 C.c_float(1e-8), self.step_n, _p(sq), C.c_float(max_norm or 0.0), _stream(p)))


class ZFilter:
    """khrylib/utils/zfilter.py ZFilter on the device: stats = [n, mean[D], S[D]] (float64)."""

    def __init__(self, dim, clip=5.0, device="cuda"):
        import torch
        self.dim, self.clip = dim, clip
        self.stats = torch.zeros(1 + 2 * dim, device=device, dtype=torch.float64)

    def __call__(self, x, update=True, out=None):
        import torch
        y = torch.empty_like(x) if out is None else out
        _chk(_lib().uhc_zfilter(_p(x), _p(y), x.shape[0], self.dim, _p(self.stats), C.c_float(self.clip), int(update), _stream(x)))
        return y

    @property
    def n(self):
        return float(self.stats[0])

    @property
    def mean(self):
        return self.stats[1:1 + self.dim].cpu().numpy()

    @property
    def std(self):
        n = self.n
        S = self.stats[1 + self.dim:].cpu().numpy()
        return np.sqrt(S / (n - 1)) if n > 1 else np.abs(self.mean)

    def load_sums(self, n, mean, S):
        """exact restore from a RunningStat's (n, mean, sum of squared deviations)"""
        import torch
        s = np.concatenate([[float(n)], np.asarray(mean, dtype=np.float64).reshape(-1), np.asarray(S, dtype=np.float64).reshape(-1)])
        self.stats.copy_(torch.as_tensor(s, dtype=torch.float64))

    def load(self, n, mean, std):
        import torch
        var = np.asarray(std, dtype=np.float64) ** 2
        s = np.concatenate([[float(n)], np.asarray(mean, dtype=np.float64), var * (max(n, 2) - 1)])
        self.stats.copy_(torch.as_tensor(s, dtype=torch.float64))


def gaussian_sample(mean, log_std, seed, step, mean_action=None, out_action=None, out_logp=None):
    import torch
    M, A = mean.shape
    a = torch.empty_like(mean) if out_action is None else out_action
    lp = torch.empty(M, device=mean.device, dtype=torch.float32) if out_logp is None else out_logp
    _chk(_lib().uhc_gaussian_sample(_p(mean), _p(log_std), _p(mean_action), _p(a), _p(lp), M, A, C.c_ulonglong(seed), C.c_ulonglong(step), _stream(mean)))
    return a, lp


def gaussian_logprob(mean, log_std, action):
    import torch
    M, A = mean.shape
    lp = torch.empty(M, device=mean.device, dtype=torch.float32)
    _chk(_lib().uhc_gaussian_logprob(_p(mean), _p(log_std), _p(action), _p(lp), M, A, _stream(mean)))
    return lp


def gae(rewards, masks, values, last_values, gamma, tau, normalize=True):
    """rewards/masks/values: [T, E] time-major.  Returns (advantages, returns), advantages normalised over the whole batch."""
    import torch
    T, E = rewards.shape
    adv, ret = torch.empty_like(rewards), torch.empty_like(rewards)
    L = _lib()
    _chk(L.uhc_gae(_p(rewards), _p(masks), _p(values), _p(last_values), C.c_float(gamma), C.c_float(tau), _p(adv), _p(ret), T, E, _stream(rewards)))
    if normalize:
        scratch = torch.zeros(2, device=rewards.device, dtype=torch.float64)
        _chk(L.uhc_normalize_advantages(_p(adv), C.c_long(adv.numel()), _p(scratch), _stream(rewards)))
    return adv, ret


class GradComm:
    """The one collective of the design (SURVEY.md section 8e): all-reduce(sum) of a net's flat gradient tensor, enqueued on a side
    stream so it overlaps the OTHER net's forward / backward; the compute stream only waits right before the optimiser step.
    Gradients arrive pre-scaled (the loss kernels divide by the GLOBAL batch size), so no division follows the collective."""

    def __init__(self, world):
        import torch
        self.world, self.torch = world, torch
        self.stream = torch.cuda.Stream() if (world > 1 and torch.cuda.is_available()) else None
        self.bytes, self.calls = 0, 0
        self.events = []

    def start(self, t):
        if self.world <= 1:
            return
        import torch.distributed as dist
        torch = self.torch
        self.bytes += t.numel() * t.element_size(); self.calls += 1
        if self.stream is None:                      # CPU / gloo (tests)
            dist.all_reduce(t)
            return
        ready = torch.cuda.current_stream().record_event()
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dist.all_reduce(t)
            e1.record()
            self.events.append((e0, e1))
        return e1

    def wait(self, done=None):
        """make the compute stream wait for one collective (its completion event) or for everything enqueued so far"""
        if self.world > 1 and self.stream is not None:
            if done is not None:
                self.torch.cuda.current_stream().wait_event(done)
            else:
                self.torch.cuda.current_stream().wait_stream(self.stream)

    def pop_ms(self):
        ms = sum(a.elapsed_time(b) for a, b in self.events)
        self.events = []
        return ms


SPLIT_CHUNKS, SPLIT_BITS, SPLIT_TOP = 5, 18, 60


def split_double(x):
    """fp64 statistics riding an fp32 all-reduce(sum) EXACTLY: x (|x| < 2^60) -> 5 float32 digit planes of 18 bits each (base 2^18
    fixed point, least significant digit = 2^-30).  Every digit is an integer below 2^18 in magnitude, so the fp32 sum over up to 32 ranks is
    exact; join_double rebuilds sum_ranks(x) to 2^-30 absolute.  Returns a [5, n] float32 tensor."""
    import torch
    r = x.to(torch.float64).clone()
    planes = []
    for k in range(SPLIT_CHUNKS):
        scale = 2.0 ** (SPLIT_TOP - SPLIT_BITS * (k + 1))
        c = torch.trunc(r / scale)
        r = r - c * scale
        planes.append(c.to(torch.float32))
    return torch.stack(planes)


def join_double(planes):
    import torch
    out = torch.zeros(planes.shape[1], dtype=torch.float64, device=planes.device)
    for k in range(SPLIT_CHUNKS):
        out = out + planes[k].to(torch.float64) * (2.0 ** (SPLIT_TOP - SPLIT_BITS * (k + 1)))
    return out


def pack_stats_tail(tail, d, extra=None):
    """the value gradient's tail for the first all-reduce of a world > 1 update: split_double's planes of the statistics d, then the extra
    payload (fp32, summed over the ranks as it is), then zeros"""
    planes = split_double(d)
    n, ne = planes.numel(), 0 if extra is None else extra.numel()
    if n + ne > tail.numel():
        raise ValueError(f"the gradient tail holds {tail.numel()} floats, the statistics and the extra payload need {n + ne}")
    tail.zero_()
    tail[:n].copy_(planes.reshape(-1))
    if ne:
        tail[n:n + ne].copy_(extra.reshape(-1))


def unpack_stats_tail(tail, nd, n_extra=0):
    """after the all-reduce: (the nd statistics summed over the ranks, fp64; the extra payload summed over the ranks, a view of the tail)"""
    n = SPLIT_CHUNKS * nd
    return join_double(tail[:n].reshape(SPLIT_CHUNKS, nd)), tail[n:n + n_extra]


def zfilter_to_sums(stats, D):
    """(n, mean, S) -> additive form (n, sum, sum of squares)"""
    import torch
    n, mean, S = stats[0:1], stats[1:1 + D], stats[1 + D:]
    return torch.cat([n, n * mean, S + n * mean * mean])


def zfilter_from_sums(sums, D):
    import torch
    n, s1, s2 = sums[0:1], sums[1:1 + D], sums[1 + D:]
    mean = s1 / torch.clamp(n, min=1.0)
    return torch.cat([n, mean, torch.clamp(s2 - n * mean * mean, min=0.0)])


def ppo_update(policy, value, log_std, opt_p, opt_v, states, actions, returns, advantages, exps, clip_eps=0.2, epochs=10, grad_clip=40.0,
               use_tc=False, comm=None):
    """AgentPPO.update_policy (agent_ppo.py:16-51), full batch: per epoch one value step then one clipped-surrogate policy step.
    use_tc=False: fp32 SIMT GEMMs (parity path); use_tc=True: wgmma bf16/fp32-accumulate GEMMs for forward, dX and dW (production)."""
    if use_tc:
        tp = getattr(policy, "_tc_trainer", None) or TCTrainer(policy)
        tv = getattr(value, "_tc_trainer", None) or TCTrainer(value)
        policy._tc_trainer, value._tc_trainer = tp, tv
        xb, xT = tp.prepare_input(states)
        tv.cache["xb"], tv.cache["xT"] = xb, xT
        return ppo_epochs_tc(policy, value, log_std, opt_p, opt_v, xb, xT, actions, returns, advantages, exps, clip_eps, epochs, grad_clip, comm=comm)
    return _ppo_update_fp32(policy, value, log_std, opt_p, opt_v, states, actions, returns, advantages, exps, clip_eps, epochs, grad_clip)


def ppo_epochs_tc(policy, value, log_std, opt_p, opt_v, xb, xT, actions, returns, advantages, exps, clip_eps=0.2, epochs=10, grad_clip=40.0,
                  comm=None, first_value=None, after_first_reduce=None, inv_count_dev=None, world=1):
    """The production update on the tensor-core path.  Per epoch: value forward/backward -> its flat gradient starts its all-reduce on the
    side stream -> policy forward / clipped-surrogate gradient / backward run meanwhile -> the policy gradient starts its all-reduce ->
    value Adam (waits for its collective) -> policy Adam.  The two nets are independent inside an epoch, so this order gives the
    reference's result (value step, then policy step, agent_ppo.py:46-51).
    first_value: (v, ctx) of a value forward already done on xb with the current weights (the V(s) GAE needed) -- reused for epoch 0.
    after_first_reduce(tail): called once the FIRST collective (value gradients + the statistics tail) is ordered before the compute
    stream: finalises everything that needs global statistics (advantage normalisation, ZFilter merge, the global row count)."""
    import torch
    L = _lib()
    tp, tv = policy._tc_trainer, value._tc_trainer
    M, A = actions.shape
    dev = actions.device
    first_policy = tp.forward(xb)                                  # old-policy mean: the fixed log-probs AND epoch 0's forward (same weights)
    fixed = gaussian_logprob(first_policy[0], log_std, actions)
    if inv_count_dev is None:
        inv_count_dev = (1.0 / torch.clamp((exps != 0).sum().to(torch.float32), min=1.0)).reshape(1)
    losses = torch.zeros(2, device=dev, dtype=torch.float32)
    comm = comm or GradComm(1)
    for ep in range(epochs):
        v, ctx = first_value if (ep == 0 and first_value is not None) else tv.forward(xb)
        dv = _buf(tv.cache, "dv", tuple(v.shape), torch.float32, dev, zero=False)
        losses.zero_()
        _chk(L.uhc_value_grad_n(_p(v), _p(returns), _p(dv), _p(losses[1:]), M, C.c_long(M * world), _stream(dv)))
        gv = tv.backward(dv, ctx, xT)
        with_tail = ep == 0 and after_first_reduce is not None
        v_done = comm.start(value.gfull if with_tail else gv)
        if with_tail:                                              # the global statistics are needed before the first policy gradient
            comm.wait(v_done)
            after_first_reduce(value.gfull[value.nflat:])
        mean, ctx = first_policy if ep == 0 else tp.forward(xb)
        dmean = _buf(tp.cache, "dmean", tuple(mean.shape), torch.float32, dev, zero=False)
        _chk(L.uhc_ppo_policy_grad_dev(_p(mean), _p(log_std), _p(actions), _p(advantages), _p(fixed), _p(exps), C.c_float(clip_eps),
                                       _p(inv_count_dev), _p(dmean), _p(losses), M, A, _stream(dmean)))
        gp = tp.backward(dmean, ctx, xT)
        p_done = comm.start(gp)
        comm.wait(v_done)                                          # value step first, as the reference; the policy collective is still in flight
        opt_v.step(gv)
        value.invalidate_bf16()
        comm.wait(p_done)
        # agent_copycat.py:93 passes `policy_net.parameters()` (a generator) as the clip list: clip_grad_norm_ exhausts it on the
        # very first call, so the reference clips only the first policy step of a run.  Mirrored here.
        first = not getattr(opt_p, "_clip_consumed", False)
        opt_p._clip_consumed = True
        opt_p.step(gp, max_norm=grad_clip if (first and grad_clip) else None)
        policy.invalidate_bf16()
    return losses


# include/uhc_ppo.h UhcAllReduceFn: ncclAllReduce's signature, the stream as a void *
ALL_REDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p)


class UhcNetDesc(C.Structure):
    """include/uhc_ppo.h UhcNetDesc"""
    _fields_ = [("nlayers", C.c_int), ("act", C.c_int), ("dims", C.c_int * 10), ("flat", C.c_void_p), ("gfull", C.c_void_p), ("nflat", C.c_long), ("gtail", C.c_long),
                ("w_off", C.c_long * 8), ("b_off", C.c_long * 8), ("adam_m", C.c_void_p), ("adam_v", C.c_void_p), ("lr", C.c_float), ("W_bf16", C.c_void_p * 8),
                ("kp", C.c_int * 8), ("head_act", C.c_int)]


class UhcPpoCfg(C.Structure):
    """include/uhc_ppo.h UhcPpoCfg"""
    _fields_ = [("gamma", C.c_float), ("tau", C.c_float), ("clip_eps", C.c_float), ("grad_clip", C.c_float), ("clip_first_step_only", C.c_int), ("epochs", C.c_int)]


def net_desc(net, opt, owner=None):
    """UhcNetDesc of an MLPNet + its flat Adam state (all pointers stay valid for the life of the net: the bf16 copies are refreshed in place).
    owner: the MCPNet whose flat tensors this sub-net lives in (offsets are then relative to the owner's tensors)."""
    if getattr(net, "_bf16_store", None) is None or net._bf16 is None:
        net._prep_bf16()
    top = owner if owner is not None else net
    assert opt.net is top, "the optimiser must be built on the net's flat tensors (nn.Adam(net.params(), lr, net=net))"
    base = net._base if owner is not None else 0
    d = UhcNetDesc()
    d.nlayers, d.act, d.head_act = len(net.W), ACT[net.htype], ACT[net.head_act]
    for i, v in enumerate(net.dims):
        d.dims[i] = v
    d.flat, d.gfull, d.nflat, d.gtail = top.flat.data_ptr(), top.gfull.data_ptr(), top.nflat, top.grad_tail
    for i in range(len(net.W)):
        d.w_off[i], d.b_off[i] = base + net._offs[2 * i][0], base + net._offs[2 * i + 1][0]
        d.W_bf16[i], d.kp[i] = net._bf16_store[i].data_ptr(), net._bf16_store[i].shape[1]
    d.adam_m, d.adam_v, d.lr = opt.mflat.data_ptr(), opt.vflat.data_ptr(), opt.lr
    d._keep = (net, opt, list(net._bf16_store))
    return d


def make_nccl_comm(rank, world, device):
    """An ncclComm_t of this process group for the C-side update (uhc_ppo_update takes the communicator, include/uhc_ppo.h): the unique id is
    made on rank 0 by the libnccl torch has loaded and broadcast through torch.distributed."""
    import torch
    import torch.distributed as dist
    lib = C.CDLL("libnccl.so.2")

    class UniqueId(C.Structure):
        _fields_ = [("internal", C.c_byte * 128)]
    uid = UniqueId()
    if rank == 0 and lib.ncclGetUniqueId(C.byref(uid)) != 0:
        raise RuntimeError("ncclGetUniqueId failed")
    t = torch.tensor(list(bytes(uid)), dtype=torch.uint8, device=device)
    dist.broadcast(t, 0)
    C.memmove(C.byref(uid), bytes(t.cpu().numpy().tobytes()), 128)
    comm = C.c_void_p()
    torch.cuda.set_device(device)
    lib.ncclCommInitRank.argtypes = [C.POINTER(C.c_void_p), C.c_int, UniqueId, C.c_int]
    if lib.ncclCommInitRank(C.byref(comm), world, uid, rank) != 0:
        raise RuntimeError("ncclCommInitRank failed")
    return comm


class CPpoTrainer:
    """uhc_ppo_update (include/uhc_ppo.h): V(s), GAE, advantage normalisation and the PPO epochs of both nets behind ONE C-ABI call, with the
    gradient all-reduce on the given ncclComm_t.  all_reduce: an ALL_REDUCE_FN the trainer calls instead of ncclAllReduce (the `comm` passed to
    update() reaches it unchanged); the trainer keeps a reference to it."""

    def __init__(self, policy, value, opt_p, opt_v, max_rows, max_envs, device, all_reduce=None):
        L = _lib()
        L.uhc_ppo_advantages.restype = C.c_void_p
        L.uhc_ppo_returns.restype = C.c_void_p
        L.uhc_ppo_kernel_launches.restype = C.c_long
        self.L, self.policy, self.value, self.opt_p, self.opt_v = L, policy, value, opt_p, opt_v
        self.dv = net_desc(value, opt_v)
        self.h = C.c_void_p()
        dev = device.index if hasattr(device, "index") else int(device)
        if isinstance(policy, MCPNet):
            arr = (UhcNetDesc * len(policy.nets))()
            self._keep = [net_desc(n, opt_p, owner=policy) for n in policy.nets]
            for i, d in enumerate(self._keep):
                arr[i] = d
            self.dp = arr
            rc = L.uhc_ppo_trainer_create_mcp(arr, C.c_int(policy.num_primitive), C.byref(self.dv), C.c_long(max_rows), C.c_int(max_envs), C.c_int(dev or 0), C.byref(self.h))
        else:
            self.dp = net_desc(policy, opt_p)
            rc = L.uhc_ppo_trainer_create(C.byref(self.dp), C.byref(self.dv), C.c_long(max_rows), C.c_int(max_envs), C.c_int(dev or 0), C.byref(self.h))
        _check(rc, "uhc_ppo_trainer_create")
        self.max_rows, self.max_envs = max_rows, max_envs
        self.all_reduce = all_reduce
        if all_reduce is not None:
            _check(L.uhc_ppo_trainer_set_all_reduce(self.h, all_reduce), "uhc_ppo_trainer_set_all_reduce")

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.L.uhc_ppo_trainer_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def update(self, states, last_states, actions, rewards, masks, exps, log_std, T, E, gamma, tau, clip_eps, epochs, grad_clip, losses, zfilter=None,
               z_sync=None, comm=None, world=1, extra_in=None, extra_out=None):
        """extra_in / extra_out: fp32 device tensors of one length whose sum over the ranks rides the first value all-reduce
        (uhc_ppo_update_ex); the value net's grad_tail must hold it behind the statistics (MLPNet.ensure_grad_tail, then a new trainer)"""
        cfg = UhcPpoCfg(gamma, tau, clip_eps, float(grad_clip or 0.0), 1, epochs)
        sp, sv = C.c_int(self.opt_p.step_n), C.c_int(self.opt_v.step_n)
        done = C.c_int(1 if getattr(self.opt_p, "_clip_consumed", False) else 0)
        n_extra = 0 if extra_in is None else extra_in.numel()
        assert n_extra == 0 or (extra_out is not None and extra_out.numel() == n_extra and extra_in.dtype == extra_out.dtype == self.policy.flat.dtype)
        rc = self.L.uhc_ppo_update_ex(self.h, _p(states), _p(last_states), _p(actions), _p(rewards), _p(masks), _p(exps), _p(log_std), C.c_int(T), C.c_int(E),
                                      C.byref(cfg), C.byref(sp), C.byref(sv), C.byref(done), _p(zfilter), _p(z_sync), comm, C.c_int(world), _p(losses),
                                      _p(extra_in), _p(extra_out), C.c_long(n_extra), _stream(states))
        _check(rc, "uhc_ppo_update")
        self.opt_p.step_n, self.opt_v.step_n = sp.value, sv.value
        self.opt_p._clip_consumed = done.value > 0
        # the C side refreshed the bf16 weight copies in place after every optimiser step
        self.policy._bf16 = getattr(self.policy, "_bf16_store", True)
        self.value._bf16 = self.value._bf16_store

    def update_policy(self, states, actions, returns, advantages, exps, log_std, clip_eps, epochs, grad_clip, losses, comm=None, world=1):
        """AgentPPO.update_policy (agent_ppo.py:16-51) on given returns / normalised advantages: uhc_ppo_update_policy"""
        cfg = UhcPpoCfg(0.0, 0.0, clip_eps, float(grad_clip or 0.0), 1, epochs)
        sp, sv = C.c_int(self.opt_p.step_n), C.c_int(self.opt_v.step_n)
        done = C.c_int(1 if getattr(self.opt_p, "_clip_consumed", False) else 0)
        rc = self.L.uhc_ppo_update_policy(self.h, _p(states), _p(actions), _p(returns), _p(advantages), _p(exps), _p(log_std), C.c_long(states.shape[0]), C.byref(cfg),
                                          C.byref(sp), C.byref(sv), C.byref(done), comm, C.c_int(world), _p(losses), _stream(states))
        _check(rc, "uhc_ppo_update_policy")
        self.opt_p.step_n, self.opt_v.step_n = sp.value, sv.value
        self.opt_p._clip_consumed = done.value > 0
        self.policy._bf16 = getattr(self.policy, "_bf16_store", True)
        self.value._bf16 = self.value._bf16_store

    @property
    def kernel_launches(self):
        return int(self.L.uhc_ppo_kernel_launches(self.h))

    def comm_stats(self):
        ms, by, calls = C.c_double(0), C.c_long(0), C.c_int(0)
        _check(self.L.uhc_ppo_comm_stats(self.h, C.byref(ms), C.byref(by), C.byref(calls)), "uhc_ppo_comm_stats")
        return ms.value, by.value, calls.value

    def advantages(self, M):
        import torch
        out = torch.empty(M, device=self.policy.flat.device, dtype=torch.float32)
        C.cdll.LoadLibrary("libcudart.so").cudaMemcpy(C.c_void_p(out.data_ptr()), C.c_void_p(self.L.uhc_ppo_advantages(self.h)), C.c_size_t(4 * M), C.c_int(3))
        return out


def _ppo_update_fp32(policy, value, log_std, opt_p, opt_v, states, actions, returns, advantages, exps, clip_eps=0.2, epochs=10, grad_clip=40.0):
    import torch
    L = _lib()
    M, A = actions.shape
    mean0 = policy.forward(states)
    fixed = gaussian_logprob(mean0, log_std, actions)
    count = float((exps != 0).sum().item())
    losses = torch.zeros(2, device=states.device, dtype=torch.float32)
    for _ in range(epochs):
        v, ctx = value.forward(states, save=True)
        dv = torch.empty_like(v)
        losses.zero_()
        _chk(L.uhc_value_grad(_p(v), _p(returns), _p(dv), _p(losses[1:]), M, _stream(states)))
        opt_v.step(value.backward(dv, ctx))
        mean, ctx = policy.forward(states, save=True)
        dmean = torch.empty_like(mean)
        _chk(L.uhc_ppo_policy_grad(_p(mean), _p(log_std), _p(actions), _p(advantages), _p(fixed), _p(exps), C.c_float(clip_eps),
                                   C.c_float(1.0 / max(count, 1.0)), _p(dmean), _p(losses), M, A, _stream(states)))
        first = not getattr(opt_p, "_clip_consumed", False)
        opt_p._clip_consumed = True
        opt_p.step(policy.backward(dmean, ctx), max_norm=grad_clip if (first and grad_clip) else None)
    policy.invalidate_bf16()
    value.invalidate_bf16()
    return losses
