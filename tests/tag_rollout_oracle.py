"""Replay oracle of the fused predator-prey rollout (ops/csrc/tag_rollout.cu).

``replay_tag_rollout`` steps ``SimpleTagEnv`` from given start positions with given standard-normal draws, using the
environment's own step, ``heuristic_prey_action`` and the PPO log-prob formula, and returns every tensor the kernel
returns in the kernel's layout.  Fed the draws ``split_rollout_marl`` makes, it reproduces that rollout bitwise on the
CPU (tests/test_tag_rollout_oracle.py); fed the kernel's draws in float64, it is the reference the GPU tests hold the
kernel to.
"""
from __future__ import annotations

import math

import torch

from nn_distributed_training_b200.rl.simple_tag import heuristic_prey_action


def log_prob(mean, act, cov_var):
    k = act.shape[-1]
    return -0.5 * ((act - mean) ** 2).sum(-1) / cov_var - 0.5 * k * math.log(2 * math.pi * cov_var)


def replay_tag_rollout(env, actors, pos0, eps, T, gamma, cov_var):
    """``pos0 [n_ep, E, A, 2]``, ``eps [N, n_ep * T * E, 5]`` (row ``(ep * T + c) * E + e``); ``actors``: one module or
    one per predator.  Returns obs, acts, log_probs, rtgs, ep_returns and the positions after every cycle
    ``pos [n_ep, T, E, A, 2]``; ``env`` is left in the last episode's final state."""
    N, E, A = env.n_adv, env.E, env.A
    n_ep = pos0.shape[0]
    nets = list(actors) if isinstance(actors, (list, tuple)) else [actors] * N
    kw = dict(device=env.device, dtype=env.dtype)
    eps = eps.to(**kw).reshape(N, n_ep, T, E, 5)
    obs_b, act_b, lp_b, rtg_b, pos_b, rets = [[] for _ in range(N)], [[] for _ in range(N)], [[] for _ in range(N)], \
        [[] for _ in range(N)], [], []
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
    cat = lambda xs: torch.stack([torch.cat(x) for x in xs])
    return dict(obs=cat(obs_b), acts=cat(act_b), log_probs=cat(lp_b), rtgs=cat(rtg_b), ep_returns=torch.cat(rets),
                pos=torch.stack(pos_b))


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
