"""A plain fp64 torch statement of what the PPO update computes, written for the tests (autograd does every derivative).

It restates the semantics the kernels implement (DESIGN.md section 5):
  - MLP / PolicyGaussian / Value / PolicyMCP forward: exact-erf GELU, tanh, relu, sigmoid after every hidden layer, a plain linear head; the
    PolicyMCP composer activates its last layer too, then a softmax weights the primitives' outputs;
  - the diagonal Gaussian log-probability, summed over the action dimension;
  - GAE by a reverse scan with masks, for one trajectory column and for a lock-step [T][E] rollout bootstrapped with V(s_T), and the
    advantage normalisation with the unbiased standard deviation;
  - the clipped surrogate over the rows with exps != 0 (torch.min of the two surrogates), the value loss mean (v - ret)^2;
  - clip_grad_norm_ and torch.optim.Adam, with the global-norm clip applied to the first policy step of a run only.
tests/test_ppo_ref.py pins it to traces of the reference's own code (tests/golden); the GPU tests compare the kernels against it.
"""
import math

import torch

F64 = torch.float64


def act(name, z):
    if name == "gelu":
        return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))
    if name == "tanh":
        return torch.tanh(z)
    if name == "relu":
        return torch.relu(z)
    if name == "sigmoid":
        return torch.sigmoid(z)
    assert name == "none", name
    return z


def mlp(params, x, htype, head_act="none", store=None):
    """params = [W0, b0, W1, b1, ...] (nn.Linear layout: W [out][in]); every layer but the last is followed by `htype`, the last by `head_act`.
    store: how the hidden activations are kept between layers (the tensor-core path keeps them in bf16); None = exactly"""
    n = len(params) // 2
    h = x
    for i in range(n):
        h = act(htype if i < n - 1 else head_act, h @ params[2 * i].t() + params[2 * i + 1])
        if store is not None and i < n - 1:
            h = store(h)
    return h


def bf16_store(h):
    """rounds the value to bf16 and passes the gradient through unchanged (what a bf16 activation buffer does to the forward pass)"""
    return h + (h.to(torch.bfloat16).to(h.dtype) - h).detach()


def mcp(prim_params, comp_params, x, htype, store=None):
    """PolicyMCP: (mean [M][A], softmax weights [M][P]) from the primitives' parameter lists and the composer's"""
    xall = torch.stack([mlp(p, x, htype, store=store) for p in prim_params], dim=1)          # [M][P][A]
    w = torch.softmax(mlp(comp_params, x, htype, head_act=htype, store=store), dim=1)
    return (w[:, :, None] * xall).sum(1), w


def mix(xall, c):
    """the mixture head alone: xall [P][M][A] primitive outputs, c [M][P] composer outputs -> (mean, softmax weights)"""
    w = torch.softmax(c, dim=1)
    return (w.t()[:, :, None] * xall).sum(0), w


def gaussian_logp(mean, log_std, actions):
    """sum over the action dimension of Normal(mean, exp(log_std)).log_prob(actions): [M]"""
    var = torch.exp(2.0 * log_std)
    return (-(actions - mean) ** 2 / (2.0 * var) - log_std - 0.5 * math.log(2.0 * math.pi)).sum(-1)


def gae_te(rewards, masks, values, gamma, tau, last_values=None):
    """lock-step rollout [T][E]: reverse scan per env column, V(s_T) = last_values (0 when None) bootstraps the last row.
    Returns the raw advantages and the returns = values + advantages."""
    T, E = rewards.shape
    dev = rewards.device
    adv = torch.zeros(T, E, dtype=F64, device=dev)
    next_v = torch.zeros(E, dtype=F64, device=dev) if last_values is None else last_values.to(F64).reshape(E)
    next_a = torch.zeros(E, dtype=F64, device=dev)
    for t in range(T - 1, -1, -1):
        delta = rewards[t] + gamma * next_v * masks[t] - values[t]
        adv[t] = delta + gamma * tau * next_a * masks[t]
        next_v, next_a = values[t], adv[t]
    return adv, values + adv


def normalize(adv):
    """(A - mean) / std with the unbiased (N - 1) standard deviation, over every element"""
    return (adv - adv.mean()) / adv.std(unbiased=True)


def estimate_advantages(rewards, masks, values, gamma, tau):
    """one trajectory column (the rows in collection order): normalised advantages and returns, both [N]"""
    adv, ret = gae_te(rewards.reshape(-1, 1), masks.reshape(-1, 1), values.reshape(-1, 1), gamma, tau)
    return normalize(adv).reshape(-1), ret.reshape(-1)


def surrogate_loss(logp, fixed_logp, adv, exps, clip_eps):
    """-mean over the rows with exps != 0 of min(r A, clip(r, 1 - eps, 1 + eps) A), r = exp(logp - fixed_logp)"""
    ind = exps.reshape(-1).nonzero().squeeze(1)
    ratio = torch.exp(logp[ind] - fixed_logp[ind])
    a = adv.reshape(-1)[ind]
    return -torch.min(ratio * a, torch.clamp(ratio, 1.0 - clip_eps, 1.0 + clip_eps) * a).mean()


def value_loss(v, ret):
    return (v.reshape(-1) - ret.reshape(-1)).pow(2).mean()


def leaves(arrays, device="cpu"):
    """fp64 leaf tensors that need gradients, from numpy arrays or tensors"""
    return [torch.as_tensor(a).detach().to(device, F64).clone().requires_grad_(True) for a in arrays]


def grads_of(loss, params):
    return [g.detach() for g in torch.autograd.grad(loss, params)]


def clip_scale(grads, max_norm):
    """the factor torch.nn.utils.clip_grad_norm_ multiplies every gradient by"""
    norm = torch.sqrt(sum((g.double() ** 2).sum() for g in grads))
    return float(torch.clamp(max_norm / (norm + 1e-6), max=1.0))


def adam(params, lr):
    return torch.optim.Adam(params, lr=lr, betas=(0.9, 0.999), eps=1e-8)


def ppo_update(pol_params, val_params, policy_mean, value_fn, log_std, states, actions, returns, advantages, exps, clip_eps, epochs, lr_p, lr_v,
               grad_clip, opt_p=None, opt_v=None, clip_done=False):
    """AgentPPO.update_policy on the full batch: per epoch one value step, then one clipped-surrogate policy step; the global-norm clip acts on
    the first policy step of a run only.  policy_mean(params, x) -> mean, value_fn(params, x) -> v.  Updates the parameters in place and returns
    (per-epoch [surrogate loss, value loss] at the weights each step saw, the policy / value gradients of the first epoch, the optimisers)."""
    opt_p = opt_p or adam(pol_params, lr_p)
    opt_v = opt_v or adam(val_params, lr_v)
    with torch.no_grad():
        fixed = gaussian_logp(policy_mean(pol_params, states), log_std, actions)
    losses, first = [], None
    for ep in range(epochs):
        lv = value_loss(value_fn(val_params, states), returns)
        opt_v.zero_grad()
        lv.backward()
        gv = [p.grad.detach().clone() for p in val_params]
        opt_v.step()
        lp = surrogate_loss(gaussian_logp(policy_mean(pol_params, states), log_std, actions), fixed, advantages, exps, clip_eps)
        opt_p.zero_grad()
        lp.backward()
        gp = [p.grad.detach().clone() for p in pol_params]
        if grad_clip and not clip_done:
            torch.nn.utils.clip_grad_norm_(pol_params, grad_clip)
            clip_done = True
        opt_p.step()
        losses.append((lp.item(), lv.item()))
        if ep == 0:
            first = (gp, gv)
    return losses, first, (opt_p, opt_v)
