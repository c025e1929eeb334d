"""float64 oracle of the PPO update kernels (ops/csrc/ppo_update.cu), written as plain functions of the weights, and
the acceptance checks that hold a kernel to it.

* ``ppo_reference`` is one node's PPO-clip actor loss and critic MSE with autograd gradients, in any dtype: float64 is
  the oracle, float32 is the torch fp32 yardstick of the fp32 kernels.  ``advantages_reference`` is the normalised
  advantage ``(A - mean) / (std + 1e-10)`` of ``A = rtgs - V`` with the unbiased std.  Both are the formulas of
  ``DistPPOProblem.ev_ppo_loss`` / ``update_advantage`` (tests/test_ppo_oracle.py holds them to it).
* ``make_batch`` draws a recorded batch that keeps every hidden pre-activation and every ratio a margin away from the
  loss's kinks, so a comparison measures rounding, not which side of a kink a sample landed on.
* ``check_fp64`` / ``check_fp32`` are the comparisons the GPU tests make; tests/test_ppo_oracle.py shows that they
  reject the defects a tiled, chunked kernel could make.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch
from torch import nn

ACT_DIM = 5
KINK_MARGIN = 1e-4   # far above the fp32 error of a pre-activation (~1e-6 of the sum of its absolute terms)
EDGE_MARGIN = 1e-3   # ratios kept this far from the clip edges 1 -+ clip
F64_LOSS, F64_GRAD = 1e-12, 1e-9   # fp64 kernels: relative error of losses / advantages and of every gradient tensor
F32_FACTOR = 4                     # fp32 kernels: at most this times the torch fp32 error ...
F32_FLOOR = 8 * torch.finfo(torch.float32).eps   # ... with a floor of a few fp32 ulps of the tensor's norm


def linears(net: nn.Module) -> List[nn.Linear]:
    return [m for m in net.seq if isinstance(m, nn.Linear)]


def weights(net: nn.Module, dtype=torch.float64):
    """``[(W_l, b_l)]`` of a ReLU MLP as detached leaf tensors of ``dtype`` that require gradients."""
    return [(m.weight.detach().to(dtype).requires_grad_(True), m.bias.detach().to(dtype).requires_grad_(True))
            for m in linears(net)]


def mlp(params, x):
    """ReLU after every layer but the last."""
    for l, (W, b) in enumerate(params):
        x = x @ W.T + b
        if l + 1 < len(params):
            x = torch.relu(x)
    return x


def log_prob(mean, act, cov_var):
    return -0.5 * ((act - mean) ** 2).sum(-1) / cov_var - 0.5 * ACT_DIM * math.log(2 * math.pi * cov_var)


def ppo_losses(actor, critic, obs, acts, old_lp, rtgs, adv, clip, cov_var, row_weight=None, open_clip=False):
    """One node's ``(actor loss, critic loss), (actor row terms, critic row terms)`` as functions of the ``weights``
    lists ``actor`` / ``critic``: ``-min(r A, clamp(r, 1 - clip, 1 + clip) A).mean()`` with ``r = exp(lp - old_lp)``
    and ``mse(V, rtgs)``.

    ``row_weight`` [R] and ``open_clip`` plant defects for tests/test_ppo_oracle.py: each row's terms are scaled by its
    weight (still divided by R), and ``open_clip`` passes the clamp's gradient on the open interval only."""
    mean = mlp(actor, obs)
    ratio = torch.exp(log_prob(mean, acts, cov_var) - old_lp)
    lo, hi = 1 - clip, 1 + clip
    if open_clip:
        inside = (ratio > lo) & (ratio < hi)
        clamped = torch.where(inside, ratio, ratio.detach().clamp(lo, hi))
    else:
        clamped = torch.clamp(ratio, lo, hi)
    a_rows = -torch.min(ratio * adv, clamped * adv)
    c_rows = (mlp(critic, obs).squeeze(-1) - rtgs) ** 2
    if row_weight is not None:
        a_rows, c_rows = row_weight * a_rows, row_weight * c_rows
    return (a_rows.mean(), c_rows.mean()), (a_rows, c_rows)


def ppo_reference(actor_net, critic_net, obs, acts, old_lp, rtgs, adv, clip, cov_var, dtype=torch.float64, **defect):
    """``(losses [2], [gradient of every parameter in actor.parameters() + critic.parameters() order], scales [2])`` of
    one node, by autograd in ``dtype`` at the nets' parameters and the given batch rows.  ``scales`` are the means of
    the losses' absolute row terms: the size of the rounding any order of summation makes."""
    actor, critic = weights(actor_net, dtype), weights(critic_net, dtype)
    cast = lambda t: t.to(dtype)                                          # noqa: E731
    (a, c), rows = ppo_losses(actor, critic, cast(obs), cast(acts), cast(old_lp), cast(rtgs), cast(adv), clip,
                              cov_var, **defect)
    leaves = [t for wb in actor + critic for t in wb]
    grads = torch.autograd.grad(a + c, leaves)
    return torch.stack([a.detach(), c.detach()]), list(grads), torch.stack([r.detach().abs().mean() for r in rows])


def gradient_scales(actor_net, critic_net, obs, acts, old_lp, rtgs, adv, clip, cov_var):
    """Per parameter tensor (``ppo_reference`` order), the float64 norm of ``sum over rows |row's gradient| / R``: the
    size of the terms every gradient sums, so of the rounding any evaluation makes when they cancel."""
    actor, critic = weights(actor_net), weights(critic_net)
    leaves = [t.detach() for wb in actor + critic for t in wb]
    na, R = 2 * len(actor), obs.shape[0]

    def row(ls, o, a, ol, rt, ad):
        pairs = lambda xs: list(zip(xs[0::2], xs[1::2]))                           # noqa: E731
        (la, lc), _ = ppo_losses(pairs(ls[:na]), pairs(ls[na:]), o[None], a[None], ol[None], rt[None], ad[None], clip,
                                 cov_var)
        return (la + lc) / R

    per_row = torch.func.vmap(torch.func.grad(row), in_dims=(None, 0, 0, 0, 0, 0))(
        leaves, *(t.double() for t in (obs, acts, old_lp, rtgs, adv)))
    return [float(g.abs().sum(0).norm()) for g in per_row]


def advantages_reference(critic_net, obs, rtgs, dtype=torch.float64, unbiased=True):
    """``(A - A.mean()) / (A.std() + 1e-10)`` of ``A = rtgs - critic(obs)`` in ``dtype``; ``unbiased=False`` plants
    the biased-std defect."""
    with torch.no_grad():
        A = rtgs.to(dtype) - mlp(weights(critic_net, dtype), obs.to(dtype)).squeeze(-1)
        return (A - A.mean()) / (A.std(unbiased=unbiased) + 1e-10)


# ---- batches --------------------------------------------------------------------------------------------------------
def near_kinks(nets_per_node: Sequence[Sequence[nn.Module]], obs, margin=KINK_MARGIN):
    """[N, R] bool: rows where a hidden pre-activation of one of node i's nets lies within ``margin`` of the ReLU
    kink, relative to the sum of the absolute values of its terms, in float64."""
    near = torch.zeros(obs.shape[:2], dtype=torch.bool, device=obs.device)
    with torch.no_grad():
        for i, nets in enumerate(nets_per_node):
            for net in nets:
                h = obs[i].double()
                for m in linears(net)[:-1]:
                    W, b = m.weight.double(), m.bias.double()
                    z = h @ W.T + b
                    near[i] |= (z.abs() < margin * (h.abs() @ W.abs().T + b.abs())).any(-1)
                    h = z.clamp_min(0)
    return near


def make_batch(actors, critics, R, clip, cov_var, seed=1, spread=0.3, kink_margin=KINK_MARGIN, device=None):
    """A recorded batch ``{obs [N, R, d0], acts [N, R, 5], log_probs [N, R], rtgs [N, R]}`` for per-node nets (lists),
    in their dtype and on their device: acts around the current actor means, so the ratios spread around 1 and some
    clip.  Rows that put a hidden pre-activation of either net within ``kink_margin`` of a ReLU kink are redrawn, and
    every ratio is moved ``EDGE_MARGIN`` away from the clip edges.  ``actors=None`` draws only obs and rtgs (the
    advantage pass, whose output is continuous in the kinks: nothing is redrawn)."""
    p = next(critics[0].parameters())
    device, dt = device or p.device, p.dtype
    N, d0 = len(critics), linears(critics[0])[0].in_features
    g = torch.Generator(device=device).manual_seed(seed)
    obs = torch.randn(N, R, d0, device=device, dtype=dt, generator=g)
    if actors is None:
        rtgs = 3.0 * torch.randn(N, R, device=device, dtype=dt, generator=g) - 1.0
        return dict(obs=obs, rtgs=rtgs)
    nets = [(a, c) for a, c in zip(actors, critics)]
    for _ in range(100 if kink_margin else 0):
        near = near_kinks(nets, obs, kink_margin)
        if not near.any():
            break
        obs = torch.where(near[..., None], torch.randn(N, R, d0, device=device, dtype=dt, generator=g), obs)
    else:
        assert not kink_margin or not near_kinks(nets, obs, kink_margin).any()
    with torch.no_grad():
        mean = torch.stack([mlp(weights(actors[i], dt), obs[i]) for i in range(N)])
    acts = mean + math.sqrt(cov_var) * torch.randn(N, R, ACT_DIM, device=device, dtype=dt, generator=g)
    lp = log_prob(mean, acts, cov_var)
    old_lp = lp + spread * torch.randn(N, R, device=device, dtype=dt, generator=g)
    r = torch.exp(lp - old_lp)
    near = ((r - (1 - clip)).abs() < EDGE_MARGIN) | ((r - (1 + clip)).abs() < EDGE_MARGIN)
    old_lp = torch.where(near, old_lp - 0.01, old_lp)     # multiplies a near-edge ratio by e^0.01
    rtgs = 3.0 * torch.randn(N, R, device=device, dtype=dt, generator=g) - 1.0
    return dict(obs=obs, acts=acts, log_probs=old_lp, rtgs=rtgs)


# ---- acceptance ------------------------------------------------------------------------------------------------------
def rel(x, ref) -> float:
    """Relative error in the 2-norm; 0 when both are zero."""
    x, ref = x.double(), ref.double()
    d = float((x - ref).norm())
    return 0.0 if d == 0.0 else d / max(float(ref.norm()), 1e-300)


def check_fp64(losses, grads, ref_losses, ref_grads, ref_scales, what="") -> float:
    """A float64 kernel's losses within ``F64_LOSS`` of the oracle, relative to the loss or, when the advantages'
    signs make the actor loss's rows cancel, to the mean absolute row term (``ref_scales``), and every gradient tensor
    within ``F64_GRAD`` (relative).  Returns the worst error as a fraction of its bound."""
    worst = 0.0
    for n in range(2):
        e = float((losses[n].double() - ref_losses[n]).abs()) / max(float(ref_losses[n].abs()), float(ref_scales[n]))
        assert e <= F64_LOSS, (what, "loss", n, e)
        worst = max(worst, e / F64_LOSS)
    for k, (g, r) in enumerate(zip(grads, ref_grads)):
        e = rel(g, r)
        assert e <= F64_GRAD, (what, "grad", k, e)
        worst = max(worst, e / F64_GRAD)
    return worst


def check_fp32(got: Sequence[torch.Tensor], ref: Sequence[torch.Tensor], *torch32: Sequence[torch.Tensor], what="",
               scales: Optional[Sequence[float]] = None) -> float:
    """Each of the float32 kernel's tensors within ``F32_FACTOR`` times the torch fp32 error against the float64
    oracle, with a floor of ``F32_FLOOR``.  ``torch32``: one or more torch fp32 evaluations of the same tensors (the
    rows summed in different orders); the yardstick is the largest of their errors, since at a few dozen rows one
    order is too narrow a sample of fp32 rounding.  ``scales``: per tensor, a size to measure the error against where
    it exceeds the reference's norm (the mean absolute row term of a loss, ``gradient_scales`` of a gradient: where
    the rows cancel, every evaluation's error is a few ulps of the terms, not of the result).  Returns the worst ratio
    of the kernel's error to the yardstick."""
    worst = 0.0
    for k, (g, r) in enumerate(zip(got, ref)):
        s = max(float(r.double().norm()), float(scales[k]) if scales is not None else 0.0, 1e-300)
        err = lambda x: float((x.double() - r.double()).norm()) / s                     # noqa: E731
        e_k, e_t = err(g), max(max(err(t[k]) for t in torch32), F32_FLOOR)
        assert e_k <= F32_FACTOR * e_t, (what, k, e_k, e_t)
        worst = max(worst, e_k / e_t)
    return worst


def check_adv64(adv, ref, what="") -> float:
    e = rel(adv, ref)
    assert e <= F64_LOSS, (what, "adv", e)
    return e / F64_LOSS


def check_losses_and_grads(dtype, losses, grads, ref, torch32=(), what="", grad_scales=None) -> float:
    """``check_fp64`` for float64 kernels, ``check_fp32`` of the losses and every gradient for float32 ones; ``ref``
    and each of ``torch32`` are ``ppo_reference`` results, ``grad_scales`` the ``gradient_scales`` (fp32)."""
    if dtype == torch.float64:
        return check_fp64(losses, grads, *ref, what)
    flat = lambda o: [o[0][0], o[0][1], *o[1]]                                        # noqa: E731
    return check_fp32(flat((losses, grads)), flat(ref), *[flat(t) for t in torch32], what=what,
                      scales=[*ref[2].tolist(), *(grad_scales or [0.0] * len(grads))])


def check_adv(dtype, adv, ref, torch32=None, what="") -> float:
    if dtype == torch.float64:
        return check_adv64(adv, ref, what)
    return check_fp32([adv], [ref], [torch32], what=what)
