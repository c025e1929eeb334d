"""Whole multi-agent PPO rollouts on the predator-prey environment as one sm_90a launch (csrc/tag_rollout.cu).

The torch path (``DistPPOProblem.split_rollout_marl``, ``PPO.rollout``, ``eval_policy.rollout``) issues about a hundred
small ops per cycle; ``rollout(...)`` runs every episode, cycle, actor forward, Gaussian action, log-prob, heuristic prey
action, contact step and reward of a batch in one kernel and returns the tensors that path collects, in its layout:
row ``(ep * T + c) * E + e`` of ``obs [N, R, obs_dim]``, ``acts [N, R, 5]``, ``log_probs [N, R]``, ``rtgs [N, R]``, and
``ep_returns [n_ep * E]``.  The actors' parameters are read in place.

The noise comes from a counter-based Philox stream keyed by ``key`` and indexed by ``index``, so it differs from the
torch path's ``randn_like`` stream; ``draw_key()`` takes the key from torch's default generator, so ``torch.manual_seed``
still determines a run.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Union

import torch
from torch import nn

from . import load_ext

MAX_AGENTS, MAX_OBSTACLES, MAX_LAYERS, MAX_WIDTH, ACT_DIM = 8, 8, 5, 64, 5


def _actor_list(env, actors) -> List[nn.Module]:
    if isinstance(actors, dict):
        return [actors[i] for i in range(env.n_adv)]
    if isinstance(actors, (list, tuple)):
        return list(actors)
    return [actors] * env.n_adv


def _linears(actor) -> Optional[List[nn.Linear]]:
    from ..models.relu_nn import FFReLUNet
    if not isinstance(actor, FFReLUNet):
        return None
    return [m for m in actor.seq if isinstance(m, nn.Linear)]


def relu_mlp_shape(nets: Sequence[nn.Module], what: str, dtype: torch.dtype):
    """``(shape, None)`` if every net is a ReLU MLP (``FFReLUNet``) with biases, parameters of ``dtype``, one common
    shape ``[d0, h1..hk, out]`` with k <= 4 hidden layers and widths <= 64 — what the sm_90a RL kernels run — and
    ``(None, reason)`` otherwise.  ``what`` names the nets in the reason ("actor", "critic")."""
    shape = None
    for a in nets:
        lin = _linears(a)
        if lin is None:
            return None, f"{what} {type(a).__name__} is not a ReLU MLP (FFReLUNet)"
        s = [lin[0].in_features] + [m.out_features for m in lin]
        if shape is not None and s != shape:
            return None, f"predators' {what}s differ in shape"
        shape = s
        if any(m.bias is None for m in lin) or any(p.dtype != dtype for p in a.parameters()):
            return None, f"{what} parameters must have biases and the dtype {dtype}"
    if not 1 <= len(shape) - 1 <= MAX_LAYERS or any(not 1 <= w <= MAX_WIDTH for w in shape):
        return None, f"{what} {shape}: needs <= {MAX_LAYERS - 1} hidden layers of width <= {MAX_WIDTH}"
    return shape, None


def unsupported_reason(env, actors) -> Optional[str]:
    """Why the kernel cannot run this environment / these actors (``None`` if it can).  The device is not checked."""
    acts = _actor_list(env, actors)
    if len(acts) != env.n_adv:
        return f"{len(acts)} actors for {env.n_adv} predators"
    if env.A > MAX_AGENTS or env.n_good < 1 or env.n_adv < 1:
        return f"needs 1..{MAX_AGENTS - 1} predators, >= 1 prey and <= {MAX_AGENTS} agents (got {env.n_adv} + {env.n_good})"
    if env.n_obs > MAX_OBSTACLES:
        return f"needs <= {MAX_OBSTACLES} obstacles"
    if env.dtype not in (torch.float32, torch.float64):
        return f"environment dtype {env.dtype} (needs float32 or float64)"
    obs_dim = env.observation_spaces["adversary_0"].shape[0]
    shape, why = relu_mlp_shape(acts, "actor", env.dtype)
    if why is not None:
        return why
    if shape[0] != obs_dim or shape[-1] != ACT_DIM:
        return f"actor {shape}: needs input {obs_dim} and output {ACT_DIM}"
    return None


def supports(env, actors) -> bool:
    """True iff the kernel covers this environment and these actors: ReLU actors ``[obs_dim, h1..hk, 5]`` with k <= 4
    and widths <= 64, at most 8 agents with at least one prey, at most 8 obstacles, float32 or float64."""
    return unsupported_reason(env, actors) is None


def require(env, actors) -> None:
    """Raise ``ValueError`` naming the reason if ``rollout`` cannot run (including a non-CUDA environment)."""
    if env.device.type != "cuda":
        raise ValueError(f"rollout backend 'cuda' needs the environment on a CUDA device (it is on {env.device})")
    why = unsupported_reason(env, actors)
    if why is not None:
        raise ValueError(f"rollout backend 'cuda' does not support this configuration: {why}")


def draw_key() -> int:
    """A 63-bit Philox key from torch's default (CPU) generator."""
    return int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())


def reset_positions(env, n_ep: int) -> torch.Tensor:
    """``pos0 [n_ep, E, A, 2]`` from ``n_ep`` ``env.reset()`` calls, in the order the torch rollout makes them."""
    out = []
    for _ in range(n_ep):
        env.reset()
        out.append(env.pos)
    return torch.stack(out)


def _distinct(env, actors):
    """The distinct actor modules and, per predator, the index of its actor among them."""
    distinct: List[nn.Module] = []
    actor_of = []
    for a in _actor_list(env, actors):
        k = next((j for j, d in enumerate(distinct) if d is a), None)
        if k is None:
            distinct.append(a)
            k = len(distinct) - 1
        actor_of.append(k)
    return distinct, actor_of


def describe(env, actors, T: int, n_ep: int, gamma: float = 1.0, cov_var: float = 1.0, noise_scale: float = 1.0,
             key: int = 0, index: int = 0, keep: Optional[list] = None) -> dict:
    """Kernel description of the actors, the environment and the episode shape, without the start positions and the
    output buffers.  Every actor parameter must be on the environment's device; non-contiguous ones are copied, and
    the copies are appended to ``keep``, which must outlive the launch."""
    require(env, actors)
    dev = env.size.device
    keep = [] if keep is None else keep

    def ptr(t):
        if t.device != dev:
            raise ValueError(f"actor parameter on {t.device}, environment on {dev}")
        t = t.detach()
        if not t.is_contiguous():
            t = t.contiguous()
            keep.append(t)
        return t.data_ptr()

    distinct, actor_of = _distinct(env, actors)
    lins = [_linears(a) for a in distinct]
    dims = [lins[0][0].in_features] + [m.out_features for m in lins[0]]
    return dict(dtype64=int(env.dtype == torch.float64), dims=dims, actor_of=actor_of,
                W=[[ptr(m.weight) for m in lin] for lin in lins], b=[[ptr(m.bias) for m in lin] for lin in lins],
                N=env.n_adv, n_good=env.n_good, A=env.A, n_obst=env.n_obs,
                size=env.size.data_ptr(), accel=env.accel.data_ptr(), max_speed=env.max_speed.data_ptr(),
                obst=env.obst.data_ptr() if env.n_obs else None,
                E=env.E, n_ep=int(n_ep), T=int(T), gamma=float(gamma), cov_var=float(cov_var),
                noise_std=float(noise_scale) * math.sqrt(cov_var),
                lp_const=0.5 * ACT_DIM * math.log(2 * math.pi * cov_var), key=int(key) & (2 ** 64 - 1),
                index=int(index) & 0xFFFFFFFF)


def launch_plan(env, actors, T: int, n_ep: int) -> Dict[str, int]:
    """The launch plan ``rollout`` would use for this environment, these actors and this episode shape on the
    environment's device, without launching: ``wpb`` worlds per CTA, ``stage`` (1: the actors are copied into shared
    memory, 0: read in place), ``rw`` worlds per register block and ``smem`` bytes of shared memory per CTA."""
    ext = load_ext(required=True)
    keep: list = []
    d = describe(env, actors, T, n_ep, keep=keep)
    with torch.cuda.device(env.size.device):
        wpb, stage, rw, smem = ext.tag_rollout_plan(d)
    return dict(wpb=wpb, stage=stage, rw=rw, smem=smem)


def rollout(env, actors, T: int, n_ep: int, gamma: float, cov_var: float, noise_scale: float = 1.0, key: int = 0,
            index: int = 0, pos0: Optional[torch.Tensor] = None, debug: bool = False,
            out: Optional[Dict[str, torch.Tensor]] = None, rews: bool = False) -> Dict[str, torch.Tensor]:
    """Run ``n_ep`` episodes of ``T`` cycles in ``env.E`` worlds each.  ``actors``: one module shared by every predator,
    or one per predator.  ``pos0`` defaults to ``reset_positions(env, n_ep)``.  Returns ``obs``, ``acts``,
    ``log_probs``, ``rtgs``, ``ep_returns`` and every world's final ``final_pos`` / ``final_vel [n_ep, E, A, 2]``;
    ``debug`` adds the standard-normal draws ``eps [N, R, 5]`` and the positions after every cycle
    ``pos [n_ep, T, E, A, 2]``.  ``rews`` adds the shared predator reward of every cycle, ``rews [N, R]`` in the batch
    layout (what generalized advantage estimation needs); ``rtgs`` is its rewards-to-go.  ``out``: contiguous tensors of the batch's shapes, dtype and device to write any of
    these into (persistent buffers); the returned dict holds them.  Afterwards ``env`` holds the last episode's final
    state, as after the torch loop (a copy, when ``out`` holds ``final_pos`` / ``final_vel``)."""
    T, n_ep = int(T), int(n_ep)
    if T < 1 or n_ep < 1:
        raise ValueError("T and n_ep must be >= 1")
    keep = []                                            # contiguous copies stay alive until the launch returns
    d = describe(env, actors, T, n_ep, gamma, cov_var, noise_scale, key, index, keep)
    ext = load_ext(required=True)
    dev, dt = env.size.device, env.dtype
    N, E, A = env.n_adv, env.E, env.A
    if pos0 is None:
        pos0 = reset_positions(env, n_ep)
    pos0 = pos0.to(device=dev, dtype=dt).contiguous()
    if tuple(pos0.shape) != (n_ep, E, A, 2):
        raise ValueError(f"pos0 has shape {tuple(pos0.shape)}, expected {(n_ep, E, A, 2)}")
    R = n_ep * T * E
    shapes = dict(obs=(N, R, d["dims"][0]), acts=(N, R, ACT_DIM), log_probs=(N, R), rtgs=(N, R), ep_returns=(n_ep * E,),
                  final_pos=(n_ep, E, A, 2), final_vel=(n_ep, E, A, 2))
    if debug:
        shapes.update(eps=(N, R, ACT_DIM), pos=(n_ep, T, E, A, 2))
    if rews:
        shapes.update(rews=(N, R))
    given = out or {}
    for k, t in given.items():
        if k not in shapes or not torch.is_tensor(t) or tuple(t.shape) != shapes[k] or t.dtype != dt \
                or t.device != dev or not t.is_contiguous():
            raise ValueError(f"out[{k!r}]: expected a contiguous {shapes.get(k)} {dt} tensor on {dev}")
    out = {k: given[k] if k in given else torch.empty(*shp, device=dev, dtype=dt) for k, shp in shapes.items()}
    d.update(pos0=pos0.data_ptr(), eps=out["eps"].data_ptr() if debug else None,
             pos_trace=out["pos"].data_ptr() if debug else None, rews=out["rews"].data_ptr() if rews else None,
             **{k: v.data_ptr() for k, v in out.items() if k not in ("eps", "pos", "rews")})
    with torch.cuda.device(dev):
        ext.tag_rollout(d)
    # the environment keeps its own copy of a caller's persistent buffer, which the next rollout into it overwrites
    final = {k: out[k][-1].clone() if k in given else out[k][-1] for k in ("final_pos", "final_vel")}
    env.pos, env.vel, env.cycle = final["final_pos"], final["final_vel"], T
    return out
