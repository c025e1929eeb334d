"""Replay oracle of the fused predator-prey rollout (ops/csrc/tag_rollout.cu).

``replay_tag_rollout`` steps ``SimpleTagEnv`` from given start positions with given standard-normal draws, using the
environment's own step, ``heuristic_prey_action`` and the PPO log-prob formula, and returns every tensor the kernel
returns in the kernel's layout.  Fed the draws ``split_rollout_marl`` makes, it reproduces that rollout bitwise on the
CPU (tests/test_tag_rollout_oracle.py); fed the kernel's draws in float64, it is the reference the GPU tests hold the
kernel to.

``check_fp64`` and ``fp32_ratio`` run the kernel and hold it to that oracle.  Contacts are stiff, so rounding
differences grow along a trajectory.  The fp64 kernel is therefore held to a yardstick: the oracle's own divergence
when ``pos0`` moves by one ulp (running max over the cycles so far, taken over all worlds); the kernel's error must
stay within 10x of it, with a floor of 1e-12 of the quantity's scale, and within 1e-12 outright on the first two
cycles.  The fp32 kernel is held to 4x the error of the torch fp32 path against the same fp64 oracle, with a floor of
a few fp32 ulps.
"""
from __future__ import annotations

import copy
import math

import torch

from nn_distributed_training_b200.ops import tag_rollout
from nn_distributed_training_b200.rl.simple_tag import SimpleTagEnv, heuristic_prey_action

GAMMA, COV = 0.99, 0.5


def log_prob(mean, act, cov_var):
    k = act.shape[-1]
    return -0.5 * ((act - mean) ** 2).sum(-1) / cov_var - 0.5 * k * math.log(2 * math.pi * cov_var)


def replay_tag_rollout(env, actors, pos0, eps, T, gamma, cov_var):
    """``pos0 [n_ep, E, A, 2]``, ``eps [N, n_ep * T * E, 5]`` (row ``(ep * T + c) * E + e``); ``actors``: one module or
    one per predator.  Returns obs, acts, log_probs, rtgs, ep_returns, the positions after every cycle
    ``pos [n_ep, T, E, A, 2]`` and every world's final velocity ``final_vel [n_ep, E, A, 2]``; ``env`` is left in the
    last episode's final state."""
    N, E, A = env.n_adv, env.E, env.A
    n_ep = pos0.shape[0]
    nets = list(actors) if isinstance(actors, (list, tuple)) else [actors] * N
    kw = dict(device=env.device, dtype=env.dtype)
    eps = eps.to(**kw).reshape(N, n_ep, T, E, 5)
    obs_b, act_b, lp_b, rtg_b, pos_b, rets = [[] for _ in range(N)], [[] for _ in range(N)], [[] for _ in range(N)], \
        [[] for _ in range(N)], [], []
    vel_b = []
    for ep in range(n_ep):
        env.pos = pos0[ep].to(**kw).clone()
        env.vel = torch.zeros(E, A, 2, **kw)
        env.cycle = 0
        obs_adv, obs_good = env.observe()
        rews, traj = [], []
        for c in range(T):
            acts = torch.zeros(E, A, 5, **kw)
            with torch.no_grad():
                for i in range(N):
                    mean = nets[i](obs_adv[:, i])
                    a = mean + math.sqrt(cov_var) * eps[i, ep, c]
                    acts[:, i] = a
                    obs_b[i].append(obs_adv[:, i]); act_b[i].append(a); lp_b[i].append(log_prob(mean, a, cov_var))
            acts[:, N:] = heuristic_prey_action(obs_good[:, 0], N).unsqueeze(1)
            r_adv, _, _ = env.step(acts)
            rews.append(r_adv)
            traj.append(env.pos.clone())
            obs_adv, obs_good = env.observe()
        R = torch.stack(rews)
        rtg = torch.zeros_like(R)
        run = torch.zeros_like(R[0])
        for s in range(R.shape[0] - 1, -1, -1):
            run = R[s] + gamma * run
            rtg[s] = run
        for i in range(N):
            rtg_b[i].append(rtg[:, :, i].reshape(-1))
        rets.append(R.sum(0).sum(-1))
        pos_b.append(torch.stack(traj))
        vel_b.append(env.vel.clone())
    cat = lambda xs: torch.stack([torch.cat(x) for x in xs])
    return dict(obs=cat(obs_b), acts=cat(act_b), log_probs=cat(lp_b), rtgs=cat(rtg_b), ep_returns=torch.cat(rets),
                pos=torch.stack(pos_b), final_vel=torch.stack(vel_b))


def draws_of_split_rollout(env, N, n_ep, T):
    """``(pos0, eps)`` drawn in the order ``split_rollout_marl`` draws them: ``env.reset()`` once per episode (from
    ``env.gen``) and ``randn_like`` once per (episode, cycle, predator) (from torch's default generator)."""
    pos0 = []
    for _ in range(n_ep):
        env.reset()
        pos0.append(env.pos.clone())
    eps = torch.empty(N, n_ep, T, env.E, 5, dtype=env.dtype)
    for ep in range(n_ep):
        for c in range(T):
            for i in range(N):
                eps[i, ep, c] = torch.randn(env.E, 5, dtype=env.dtype)
    return torch.stack(pos0), eps.reshape(N, n_ep * T * env.E, 5)


# ---- the kernel against the oracle (GPU) -----------------------------------------------------------------------------
def tag_env(E=16, n_adv=3, n_good=1, n_obst=8, max_cycles=200, dtype=torch.float64, device="cuda", seed=0):
    return SimpleTagEnv(num_envs=E, num_good=n_good, num_adversaries=n_adv, num_obstacles=n_obst, max_cycles=max_cycles,
                        device=device, dtype=dtype, seed=seed)


def on(actors, device):
    """Copies of ``actors`` (a list) on ``device``; entries that are the same module stay one module."""
    memo = {}
    return [memo.setdefault(id(a), copy.deepcopy(a).to(device)) for a in actors]


def _per_cycle(x, n_ep, T, E):
    """[N, R, ...] -> [T, everything else] (max over worlds is taken per cycle)."""
    N = x.shape[0]
    return x.reshape(N, n_ep, T, E, -1).permute(2, 0, 1, 3, 4).reshape(T, -1)


def _cycles(out, n_ep, T, E):
    q = {k: _per_cycle(out[k].double().cpu(), n_ep, T, E) for k in ("obs", "acts", "log_probs", "rtgs")}
    q["pos"] = out["pos"].double().cpu().permute(1, 0, 2, 3, 4).reshape(T, -1)
    return q


def _err(a, b):
    return {k: (a[k] - b[k]).abs().amax(dim=1) for k in a}            # [T] per quantity


def _envelope(e):
    return torch.cummax(e, dim=0).values


def run_kernel(env, actors, pos0, T, key=7, index=0, noise=1.0, out=None):
    n_ep = pos0.shape[0]
    res = tag_rollout.rollout(env, actors, T=T, n_ep=n_ep, gamma=GAMMA, cov_var=COV, noise_scale=noise, key=key,
                              index=index, pos0=pos0, debug=True, out=out)
    torch.cuda.synchronize()
    return res


def oracle(actors, pos0, eps, T, cfg, dtype=torch.float64):
    env = tag_env(**dict(cfg, dtype=dtype, device="cpu"))
    acts = [a.to("cpu", dtype) for a in on(actors, "cpu")]
    return replay_tag_rollout(env, acts, pos0.to("cpu", dtype), eps.to("cpu", dtype), T, GAMMA, COV)


def _check_final(out, ref, yard, factor, floor_rel):
    """Every world's final position is its position after the last cycle, bit for bit; its final velocity is held to
    ``factor`` times the yardstick's error in the velocity or in the positions (a velocity error e moves the next
    position by 0.1 e, so 10x the position error), with a floor of ``floor_rel`` of the scale."""
    assert torch.equal(out["final_pos"], out["pos"][:, -1])
    vk, vo, vy = out["final_vel"].double().cpu(), ref["final_vel"], yard["final_vel"]
    ey = max((vy - vo).abs().max().item(), 10 * (yard["pos"] - ref["pos"]).abs().max().item())
    bound = max(factor * ey, floor_rel * max(vo.abs().max().item(), 1.0))
    assert (vk - vo).abs().max().item() <= bound, ("final_vel", (vk - vo).abs().max().item(), bound)


def check_fp64(cfg, actors, n_ep, T, out=None):
    """Run the fp64 kernel on ``tag_env(**cfg)`` from ``reset_positions`` and hold every output to the oracle;
    ``out``: buffers for ``rollout``.  Returns the outputs and the worst error as a fraction of its bound."""
    env = tag_env(**cfg)
    pos0 = tag_rollout.reset_positions(env, n_ep)
    res = run_kernel(env, actors, pos0, T, out=out)
    E = env.E
    ref = oracle(actors, pos0, res["eps"], T, cfg)
    up = torch.nextafter(pos0.cpu(), torch.tensor(float("inf"), dtype=torch.float64))
    yard = oracle(actors, up, res["eps"], T, cfg)
    k, o, y = _cycles(res, n_ep, T, E), _cycles(ref, n_ep, T, E), _cycles(yard, n_ep, T, E)
    ek, ey = _err(k, o), _err(y, o)
    worst = 0.0
    for q in k:
        scale = o[q].abs().max().item()
        bound = torch.clamp(10 * _envelope(ey[q]), min=1e-12 * scale)
        assert (ek[q] <= bound).all(), (q, ek[q].tolist(), bound.tolist())
        if q != "rtgs":                                   # an early reward-to-go sums the whole episode
            assert (ek[q][:2] <= 1e-12 * max(scale, 1.0)).all(), (q, ek[q][:2].tolist())
        worst = max(worst, (ek[q] / bound).max().item())
    rk, ro, ry = res["ep_returns"].cpu(), ref["ep_returns"], yard["ep_returns"]
    assert (rk - ro).abs().max() <= max(10 * (ry - ro).abs().max().item(), 1e-12 * ro.abs().max().item())
    _check_final(res, ref, yard, 10, 1e-12)
    print(f"fp64 kernel error / bound, worst over quantities and cycles: {worst:.3g}")
    return res, worst


def fp32_ratio(cfg, actors32, T, n_ep, noise=1.0, perturbed_yardstick=False, out=None):
    """Run the fp32 kernel and hold every output to 4x the torch fp32 error against the fp64 oracle.
    ``perturbed_yardstick``: the torch fp32 error is the larger of the runs from pos0 and from pos0 moved by one fp32
    ulp.  The deterministic trained policy keeps the predators in stiff contact, so when the trajectories first
    amplify a rounding difference depends on where that difference lands; one torch run is then too narrow a sample.
    Returns the outputs and the worst ratio of the kernel's error to the torch fp32 error."""
    env = tag_env(**dict(cfg, dtype=torch.float32))
    pos0 = tag_rollout.reset_positions(env, n_ep)
    res = run_kernel(env, actors32, pos0, T, noise=noise, out=out)
    E = env.E
    eps = res["eps"] * noise
    ref = oracle(actors32, pos0, eps, T, cfg)                                         # fp64 oracle, fp32 inputs
    t32 = oracle(actors32, pos0, eps, T, cfg, dtype=torch.float32)                    # the torch fp32 path
    k, o, t = _cycles(res, n_ep, T, E), _cycles(ref, n_ep, T, E), _cycles(t32, n_ep, T, E)
    ek, et = _err(k, o), _err(t, o)
    if perturbed_yardstick:
        up = torch.nextafter(pos0.cpu(), torch.tensor(float("inf")))
        t2 = _cycles(oracle(actors32, up, eps, T, cfg, dtype=torch.float32), n_ep, T, E)
        et = {q: torch.maximum(et[q], v) for q, v in _err(t2, o).items()}
    worst = 0.0
    for q in k:
        scale = o[q].abs().max().item()
        floor = 4 * 2.0 ** -23 * scale
        bound = torch.clamp(4 * _envelope(et[q]), min=floor)
        assert (ek[q] <= bound).all(), (q, ek[q].tolist(), bound.tolist())
        worst = max(worst, (ek[q] / torch.clamp(_envelope(et[q]), min=floor)).max().item())
    _check_final(res, ref, t32, 4, 4 * 2.0 ** -23)
    print(f"fp32 kernel error / torch fp32 error, worst over quantities and cycles: {worst:.3g}")
    return res, worst
