"""The PPO update on sm_90a (csrc/ppo_update.cu): per-node advantages and every node's actor and critic gradients.

The torch path (``DistPPOProblem.evaluate`` / ``ev_ppo_loss`` and autograd, ``PPO.learn``) runs about fifty launches and
one host synchronisation per node per primal step.  Here

* ``advantages(critics, obs, rtgs)`` is the critic forward over every node's samples and the per-node normalisation
  ``(A - mean) / (std + 1e-10)`` of ``A = rtgs - V`` (two launches); with ``gae=GAE(...)`` ``A`` is the GAE(lambda)
  advantage of the per-cycle rewards and the lambda-returns ``A + V`` come back as the critic's target (three
  launches), and
* ``grads(...)`` is one primal step of every node: forward, PPO-clip actor loss, critic MSE and both backward passes,
  written straight into the caller's gradient tensors (two launches, no synchronisation).

The batch layout is the rollout kernel's: node ``i``'s samples are row ``i`` of ``obs [N, R, obs_dim]``,
``acts [N, R, 5]`` and ``old_lp / rtgs / adv [N, R]``.  The networks' parameters are read in place.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch import nn

from . import load_ext
from .tag_rollout import ACT_DIM, _linears, relu_mlp_shape

MAX_NODES = 8


def _as_list(nets) -> List[nn.Module]:
    if isinstance(nets, dict):
        return [nets[i] for i in range(len(nets))]
    if isinstance(nets, (list, tuple)):
        return list(nets)
    return [nets]


def unsupported_reason(actors, critics) -> Optional[str]:
    """Why the kernels cannot run these per-node actors / critics (``None`` if they can).  The device is not checked:
    ReLU MLPs (``FFReLUNet``) with biases, ``[obs_dim, h1..hk, 5]`` actors and ``[obs_dim, h1..hk, 1]`` critics with
    k <= 4 and widths <= 64, float32 or float64, 1..8 nodes.  ``actors=None`` checks the critics alone (the advantage
    pass)."""
    crits = _as_list(critics)
    acts = _as_list(actors) if actors is not None else None
    if (acts is not None and len(acts) != len(crits)) or not 1 <= len(crits) <= MAX_NODES:
        got = f"{len(acts)} and {len(crits)}" if acts is not None else f"{len(crits)} critics"
        return f"needs 1..{MAX_NODES} nodes with one actor and one critic each (got {got})"
    p = next(crits[0].parameters(), None)
    dtype = p.dtype if p is not None else None
    if dtype not in (torch.float32, torch.float64):
        return f"parameter dtype {dtype} (needs float32 or float64)"
    sc, why = relu_mlp_shape(crits, "critic", dtype)
    if why is not None:
        return why
    if sc[-1] != 1:
        return f"critic {sc}: needs output 1"
    if acts is None:
        return None
    sa, why = relu_mlp_shape(acts, "actor", dtype)
    if why is not None:
        return why
    if sa[-1] != ACT_DIM:
        return f"actor {sa}: needs output {ACT_DIM}"
    if sa[0] != sc[0]:
        return f"actor {sa} / critic {sc}: input widths differ"
    return None


def supports(actors, critics) -> bool:
    """True iff the kernels cover these actors and critics (see ``unsupported_reason``)."""
    return unsupported_reason(actors, critics) is None


def require(actors, critics) -> None:
    """Raise ``ValueError`` naming the reason if the kernels cannot run (including parameters not on a CUDA device).
    ``actors=None`` checks the critics alone."""
    for m in (_as_list(actors) if actors is not None else []) + _as_list(critics):
        for p in m.parameters():
            if p.device.type != "cuda":
                raise ValueError(f"update backend 'cuda' needs the networks on a CUDA device (a parameter is on {p.device})")
    why = unsupported_reason(actors, critics)
    if why is not None:
        raise ValueError(f"update backend 'cuda' does not support this configuration: {why}")


def _desc(actors, critics, dtype, dev, N, R):
    """Kernel description of N (actor, critic) pairs whose parameters are on ``dev``; ``actors=None`` describes the
    critics only."""
    crits = _as_list(critics)
    acts = _as_list(actors) if actors is not None else []
    if len(crits) != N or (actors is not None and len(acts) != N):
        raise ValueError(f"{len(acts)} actors and {len(crits)} critics for a batch of {N} nodes")
    for m in acts + crits:
        for p in m.parameters():
            if p.device != dev:
                raise ValueError(f"network parameter on {p.device}, batch on {dev}")
            if p.dtype != dtype or not p.is_contiguous():
                raise ValueError(f"network parameters must be contiguous CUDA tensors of the batch dtype {dtype}")
    lins = [[_linears(a) if actors is not None else [], _linears(c)] for a, c in zip(acts or [None] * N, crits)]
    dims = [[ln[0].in_features] + [m.out_features for m in ln] if ln else [] for ln in lins[0]]
    return dict(dtype64=int(dtype == torch.float64), N=N, R=R, dims=dims,
                W=[[[m.weight.data_ptr() for m in ln] for ln in node] for node in lins],
                b=[[[m.bias.data_ptr() for m in ln] for ln in node] for node in lins], clip=0.0, cov_var=1.0, lp_const=0.0)


def _described(t) -> str:
    """``t``'s shape, dtype and device as an error message shows them (a device inside a tuple would print as
    ``device(type='cuda', index=1)``)."""
    return f"{tuple(t.shape)} {t.dtype} on {t.device}" if torch.is_tensor(t) else type(t).__name__


def _batch(name, t, shape, dtype, dev):
    if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape) or t.dtype != dtype or t.device != dev:
        got = _described(t)
        raise ValueError(f"{name}: expected {tuple(shape)} {dtype} on {dev}, got {got}")
    return t.contiguous()


@dataclass
class GAE:
    """Generalized advantage estimation for ``advantages``: ``rews [N, R]`` the per-cycle rewards in the batch's row
    order ``r = (blk * T + c) * E + e`` (``T`` cycles of ``E`` worlds per block, ``T * E`` dividing ``R``; each block
    ends in a terminal step), discount ``gamma`` and ``lam`` in [0, 1].  ``returns``: an optional contiguous
    ``[N, R]`` output for the lambda-returns; ``values``: an optional one the critic's ``V`` is copied into (the
    baseline the advantages subtract, for diagnostics such as the explained variance)."""
    rews: torch.Tensor
    gamma: float
    lam: float
    T: int
    E: int
    returns: Optional[torch.Tensor] = None
    values: Optional[torch.Tensor] = None


def advantages(critics, obs: torch.Tensor, rtgs: torch.Tensor, out: Optional[torch.Tensor] = None, *,
               gae: Optional[Union[GAE, dict]] = None) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]:
    """``[N, R]`` normalised advantages ``(A - mean) / (std + 1e-10)`` of ``A = rtgs - critic_i(obs[i])``, with node
    ``i``'s mean and unbiased std (so NaN for R = 1, as torch's ``std``).  ``critics``: one per node.  ``out``: a
    contiguous ``[N, R]`` tensor of the batch dtype to write them into (returned).

    ``gae``: a ``GAE`` (or a dict of its fields).  Then ``A`` is the GAE(lambda) advantage of ``gae.rews`` within each
    (episode block, world), ``delta_c = r_c + gamma V_{c+1} - V_c`` and ``A_c = delta_c + gamma lam A_{c+1}`` with
    ``V_T = A_T = 0``, and the call returns ``(adv, returns)``: ``returns = A + V`` is the critic's target, written into
    ``gae.returns`` when given.  ``rtgs`` then does not enter the result."""
    crits = _as_list(critics)
    require(None, crits)
    ext = load_ext(required=True)
    if rtgs.dim() != 2:
        raise ValueError(f"rtgs: expected [N, R], got {tuple(rtgs.shape)}")
    N, R = rtgs.shape
    dev, dt = rtgs.device, rtgs.dtype
    d = _desc(None, crits, dt, dev, N, R)
    obs = _batch("obs", obs, (N, R, d["dims"][1][0]), dt, dev)
    rtgs = rtgs.contiguous()
    adv = torch.empty(N, R, device=dev, dtype=dt) if out is None else _out("out", out, (N, R), dt, dev)
    d.update(obs=obs.data_ptr(), rtgs=rtgs.data_ptr(), adv=adv.data_ptr())
    if gae is not None:
        g = GAE(**gae) if isinstance(gae, dict) else gae
        T, E, gamma, lam = int(g.T), int(g.E), float(g.gamma), float(g.lam)
        if T < 1 or E < 1 or R % (T * E):
            raise ValueError(f"gae: T * E = {T} * {E} must divide R = {R}")
        if not (0.0 <= gamma <= 1.0 and 0.0 <= lam <= 1.0):
            raise ValueError(f"gae: gamma {gamma} and lam {lam} must lie in [0, 1]")
        rews = _batch("gae.rews", g.rews, (N, R), dt, dev)
        ret = torch.empty(N, R, device=dev, dtype=dt) if g.returns is None \
            else _out("gae.returns", g.returns, (N, R), dt, dev)
        vals = None if g.values is None else _out("gae.values", g.values, (N, R), dt, dev).data_ptr()
        d.update(gae=True, T=T, E=E, gamma=gamma, lam=lam, rews=rews.data_ptr(), returns=ret.data_ptr(), values=vals)
    with torch.cuda.device(dev):
        ext.ppo_advantages(d)
    return adv if gae is None else (adv, ret)


def launch_plan(actors, critics, R: int, backward: bool = True) -> Dict[str, int]:
    """The launch plan of ``grads`` (``backward=True``) or of ``advantages`` (``backward=False``, ``actors`` unused)
    for these per-node networks and ``R`` samples per node on the networks' device, without launching: ``tm`` rows per
    tile, ``chunks`` CTAs per node and network (each walks ``per = ceil(ceil(R / chunks) / tm) * tm`` rows),
    ``smem`` bytes of dynamic shared memory per CTA and ``work_bytes`` of workspace (the partial-sum slots of
    ``grads``; 0 for ``advantages``)."""
    crits = _as_list(critics)
    acts = _as_list(actors) if backward else None
    require(acts, crits)
    ext = load_ext(required=True)
    p = next(crits[0].parameters())
    d = _desc(acts, crits, p.dtype, p.device, len(crits), int(R))
    with torch.cuda.device(p.device):
        tm, chunks, smem, work_bytes = ext.ppo_plan(d, bool(backward))
    return dict(tm=tm, chunks=chunks, smem=smem, work_bytes=work_bytes)


def _out(name, t, shape, dtype, dev):
    """An output tensor the kernel writes in place: exactly ``shape``, ``dtype``, ``dev`` and contiguous."""
    if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape) or t.dtype != dtype or t.device != dev \
            or not t.is_contiguous():
        got = _described(t)
        raise ValueError(f"{name}: expected a contiguous {tuple(shape)} {dtype} tensor on {dev}, got {got}")
    return t


# Network and gradient descriptions already validated, keyed by every parameter's and gradient tensor's address and
# shape: a primal step re-validates nothing unless a tensor moved.
_DESCS: Dict[tuple, dict] = {}


def _grads_desc(acts_l, crits, grad_out, N, R, dt, dev):
    params = [list(a.parameters()) + list(c.parameters()) for a, c in zip(acts_l, crits)]
    key = (N, R, dt, dev, tuple(type(m) for m in acts_l + crits),
           tuple((p.data_ptr(), p.shape) for node in params for p in node),
           tuple((t.data_ptr(), t.shape, t.dtype) for node in grad_out for t in node))
    d = _DESCS.get(key)
    if d is not None:
        return d
    require(acts_l, crits)
    d = _desc(acts_l, crits, dt, dev, N, R)
    gW, gb = [], []
    for i in range(N):
        g = list(grad_out[i])
        if len(g) != len(params[i]):
            raise ValueError(f"grad_out[{i}]: {len(g)} tensors for {len(params[i])} parameters")
        for p, t in zip(params[i], g):
            if t.shape != p.shape or t.dtype != dt or t.device != dev or not t.is_contiguous():
                raise ValueError(f"grad_out[{i}]: expected contiguous {tuple(p.shape)} {dt} tensors on {dev}, "
                                 f"got {_described(t)}")
        na = len(list(acts_l[i].parameters()))
        gW.append([[t.data_ptr() for t in g[:na:2]], [t.data_ptr() for t in g[na::2]]])
        gb.append([[t.data_ptr() for t in g[1:na:2]], [t.data_ptr() for t in g[na + 1::2]]])
    d.update(gW=gW, gb=gb)
    if len(_DESCS) >= 16:
        _DESCS.clear()
    _DESCS[key] = d
    return d


def grads(actors, critics, obs: torch.Tensor, acts: torch.Tensor, old_lp: torch.Tensor, rtgs: torch.Tensor,
          adv: torch.Tensor, clip: float, cov_var: float, grad_out: Sequence[Sequence[torch.Tensor]],
          nonfinite: Optional[torch.Tensor] = None, losses_out: Optional[torch.Tensor] = None,
          workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One primal step of every node: writes the gradients of node ``i``'s PPO-clip actor loss and critic MSE into
    ``grad_out[i]`` — one tensor per parameter, in ``parameters()`` order of the actor then the critic (arena-row views
    or ``p.grad``) — and returns ``losses [N, 2]`` (actor, critic), written into ``losses_out`` when given (a
    contiguous ``[N, 2]`` tensor of the batch dtype, for example a row of a buffer a CUDA graph replays into).
    ``nonfinite``, an int32 CUDA tensor, is set to 1 if an actor mean is not finite; it is never cleared here.
    ``workspace``: a contiguous, 16-byte aligned uint8 tensor on the batch's device of at least ``launch_plan(...)["work_bytes"]``
    bytes for the per-CTA partial sums (default: one from the caching allocator per call).  Nothing is synchronised."""
    acts_l, crits = _as_list(actors), _as_list(critics)
    ext = load_ext(required=True)
    if rtgs.dim() != 2:
        raise ValueError(f"rtgs: expected [N, R], got {tuple(rtgs.shape)}")
    N, R = rtgs.shape
    dev, dt = rtgs.device, rtgs.dtype
    if len(acts_l) != N or len(crits) != N or len(grad_out) != N:
        raise ValueError(f"{len(acts_l)} actors, {len(crits)} critics and {len(grad_out)} gradient lists for {N} nodes")
    d = dict(_grads_desc(acts_l, crits, grad_out, N, R, dt, dev))
    obs = _batch("obs", obs, (N, R, d["dims"][0][0]), dt, dev)
    acts = _batch("acts", acts, (N, R, ACT_DIM), dt, dev)
    old_lp = _batch("old_lp", old_lp, (N, R), dt, dev)
    adv = _batch("adv", adv, (N, R), dt, dev)
    rtgs = rtgs.contiguous()
    losses = torch.empty(N, 2, device=dev, dtype=dt) if losses_out is None else _out("losses_out", losses_out, (N, 2), dt, dev)
    if nonfinite is None:
        nonfinite = torch.zeros(1, device=dev, dtype=torch.int32)
    elif nonfinite.dtype != torch.int32 or nonfinite.device != dev:
        raise ValueError(f"nonfinite: expected an int32 tensor on {dev}")
    d.update(obs=obs.data_ptr(), acts=acts.data_ptr(), old_lp=old_lp.data_ptr(), rtgs=rtgs.data_ptr(),
             adv=adv.data_ptr(), clip=float(clip), cov_var=float(cov_var),
             lp_const=0.5 * ACT_DIM * math.log(2 * math.pi * cov_var), losses=losses.data_ptr(),
             nonfinite=nonfinite.data_ptr())
    if workspace is not None:
        if workspace.dtype != torch.uint8 or workspace.device != dev or not workspace.is_contiguous() \
                or workspace.data_ptr() % 16:
            raise ValueError(f"workspace: expected a contiguous, 16-byte aligned uint8 tensor on {dev}, "
                             f"got {_described(workspace)}")
        d.update(work=workspace.data_ptr(), work_bytes=workspace.numel())
    with torch.cuda.device(dev):
        ext.ppo_grads(d)
    return losses
