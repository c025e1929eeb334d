"""Multi-agent PPO as a distributed-learning problem (reference: RL/dist_rl/dist_ppo.py:19-491).

Each graph node is one predator with its own actor/critic pair; nodes share nothing but the
consensus updates.  Rollouts come from the batched ``SimpleTagEnv`` (``num_envs`` worlds stepped
together, one actor forward per predator per cycle for the whole batch) instead of the
reference's one-agent-at-a-time Python loop, and the problem exposes the reference problem API
(``N, graph, models, local_batch_loss(i), update_graph(), evaluate_metrics()``) so the generic
arena-based DiNNO / DSGD / DSGT drive it unchanged.
"""
from __future__ import annotations

import copy
import math
import time
from typing import Dict

import numpy as np
import torch
from torch import nn

from .model import ActorCritic
from .simple_tag import SimpleTagEnv, heuristic_prey_action


class DistPPOProblem:
    # defaults of the reference's _init_hyperparameters (:391-436) — set explicitly, no exec()
    # rollout_backend "cuda": each batch is one fused kernel launch (ops/tag_rollout.py) with its own Philox noise stream
    DEFAULTS = dict(timesteps_per_batch=4800, max_timesteps_per_episode=1600, n_updates_per_iteration=5,
                    lr=0.005, gamma=0.95, clip=0.2, render=False, render_every_i=10, save_freq=10, seed=None,
                    rollout_backend="torch")

    def __init__(self, base_actor, base_critic, graph, env: SimpleTagEnv, **hyperparameters):
        for k, v in {**self.DEFAULTS, **hyperparameters}.items():
            if k not in self.DEFAULTS:
                raise TypeError(f"unknown PPO hyper-parameter {k!r}")
            setattr(self, k, v)
        if self.seed is not None:
            assert isinstance(self.seed, int)
            torch.manual_seed(self.seed)
            print(f"Successfully set seed to {self.seed}")
        self.env = env
        self.obs_dim = env.observation_spaces["adversary_0"].shape[0]
        self.act_dim = env.action_spaces["adversary_0"].shape[0]
        self.graph = graph
        self.N = graph.number_of_nodes()
        if self.N != env.n_adv:
            raise ValueError("one graph node per predator")
        self.device = env.device
        self.models: Dict[int, ActorCritic] = {}
        for i in range(self.N):
            m = ActorCritic.__new__(ActorCritic)
            nn.Module.__init__(m)
            m.actor, m.critic = copy.deepcopy(base_actor), copy.deepcopy(base_critic)
            self.models[i] = m.to(self.device)
        self.n_actor = sum(p.numel() for p in base_actor.parameters())
        self.n_critic = sum(p.numel() for p in base_critic.parameters())
        self.cov_var = 0.5                       # fixed diagonal covariance (:66-67)
        self.conf = {"metrics_config": {"evaluate_frequency": 10 ** 12}, "problem_name": "dist_ppo"}
        self.logger = {"delta_t": time.time_ns(), "t_so_far": 0, "i_so_far": 0, "batch_lens": [],
                       "batch_rews": [], "actor_losses": []}
        if self.rollout_backend not in ("torch", "cuda"):
            raise ValueError(f"rollout_backend must be 'torch' or 'cuda', not {self.rollout_backend!r}")
        if self.rollout_backend == "cuda":
            from ..ops import tag_rollout
            tag_rollout.require(env, self.actors)
        self._rollout_key, self._rollout_index = None, 0

    @property
    def actors(self):
        return {i: m.actor for i, m in self.models.items()}

    @property
    def critics(self):
        return {i: m.critic for i, m in self.models.items()}

    # ---- policy ---------------------------------------------------------------------
    def _log_prob(self, mean, act):
        k = act.shape[-1]
        return -0.5 * ((act - mean) ** 2).sum(-1) / self.cov_var - 0.5 * k * math.log(2 * math.pi * self.cov_var)

    def get_action(self, i, obs):
        """Sample a ~ N(actor_i(obs), 0.5 I); returns (action, log_prob), both detached."""
        with torch.no_grad():
            mean = self.models[i].actor(obs)
            act = mean + math.sqrt(self.cov_var) * torch.randn_like(mean)
            return act, self._log_prob(mean, act)

    def evaluate(self, i):
        V = self.models[i].critic(self.curr_obs[i]).squeeze(-1)
        mean = self.models[i].actor(self.curr_obs[i])
        if not torch.isfinite(mean).all():
            raise NameError("actor returning something weird")
        return V, self._log_prob(mean, self.curr_acts[i])

    # ---- data collection ---------------------------------------------------------------
    def split_rollout_marl(self):
        """Collect at least ``timesteps_per_batch`` predator steps (ALG STEP 3)."""
        if self.rollout_backend == "cuda":
            return self._split_rollout_cuda()
        env, N = self.env, self.N
        cycles = max(1, self.max_timesteps_per_episode // env.num_agents)
        obs_b = [[] for _ in range(N)]; act_b = [[] for _ in range(N)]
        lp_b = [[] for _ in range(N)]; rtg_b = [[] for _ in range(N)]
        ep_returns, ep_lens, t = [], [], 0
        while t < self.timesteps_per_batch:
            obs_adv, obs_good = env.reset()
            rews = []
            for c in range(cycles):
                acts = torch.zeros(env.E, env.A, 5, device=self.device, dtype=obs_adv.dtype)
                for i in range(N):
                    a, lp = self.get_action(i, obs_adv[:, i])
                    acts[:, i] = a
                    obs_b[i].append(obs_adv[:, i]); act_b[i].append(a); lp_b[i].append(lp)
                acts[:, N:] = heuristic_prey_action(obs_good[:, 0], env.n_adv).unsqueeze(1)
                r_adv, _, done = env.step(acts)
                rews.append(r_adv)
                obs_adv, obs_good = env.observe()
                t += N * env.E
                if done:
                    break
            R = torch.stack(rews)                                  # [T, E, N]
            rtg = torch.zeros_like(R)
            run = torch.zeros_like(R[0])
            for s in range(R.shape[0] - 1, -1, -1):                 # rewards-to-go (ALG STEP 4)
                run = R[s] + self.gamma * run
                rtg[s] = run
            for i in range(N):
                rtg_b[i].append(rtg[:, :, i])
            ep_returns.extend(R.sum(0).sum(-1).tolist())            # joint predator return per world
            ep_lens.extend([R.shape[0] * env.num_agents] * env.E)
        flat = lambda xs: torch.cat([x.reshape(-1, *x.shape[2:]) if x.dim() > 2 else x.reshape(-1) for x in xs])
        self.curr_obs = {i: torch.cat(obs_b[i]) for i in range(N)}
        self.curr_acts = {i: torch.cat(act_b[i]) for i in range(N)}
        self.curr_log_probs = {i: torch.cat(lp_b[i]) for i in range(N)}
        self.curr_rtgs = {i: torch.cat([r.reshape(-1) for r in rtg_b[i]]) for i in range(N)}
        self.logger["batch_rews"] = ep_returns
        self.logger["batch_lens"] = ep_lens
        self.logger["t_so_far"] += int(np.sum(ep_lens))
        self.logger["i_so_far"] += 1

    def _split_rollout_cuda(self):
        """The same batch as ``split_rollout_marl`` (episodes, cycles, layout, counts) from one kernel launch."""
        from ..ops import tag_rollout
        env, N = self.env, self.N
        T = min(max(1, self.max_timesteps_per_episode // env.num_agents), env.max_cycles)
        n_ep = max(1, -(-self.timesteps_per_batch // (N * env.E * T)))
        if self._rollout_key is None:
            self._rollout_key = tag_rollout.draw_key()
        out = tag_rollout.rollout(env, self.actors, T=T, n_ep=n_ep, gamma=self.gamma, cov_var=self.cov_var,
                                  key=self._rollout_key, index=self._rollout_index)
        self._rollout_index += 1
        self.curr_obs = {i: out["obs"][i] for i in range(N)}
        self.curr_acts = {i: out["acts"][i] for i in range(N)}
        self.curr_log_probs = {i: out["log_probs"][i] for i in range(N)}
        self.curr_rtgs = {i: out["rtgs"][i] for i in range(N)}
        ep_lens = [T * env.num_agents] * (n_ep * env.E)
        self.logger["batch_rews"] = out["ep_returns"].tolist()
        self.logger["batch_lens"] = ep_lens
        self.logger["t_so_far"] += int(np.sum(ep_lens))
        self.logger["i_so_far"] += 1

    def compute_rtgs(self, batch_rews):
        out = []
        for ep in reversed(batch_rews):
            d = 0.0
            for r in reversed(ep):
                d = r + d * self.gamma
                out.insert(0, d)
        return torch.tensor(out, dtype=torch.float)

    def update_advantage(self):
        self.A_k = {}
        with torch.no_grad():
            for i in range(self.N):
                V, _ = self.evaluate(i)
                A = self.curr_rtgs[i] - V                             # ALG STEP 5
                self.A_k[i] = (A - A.mean()) / (A.std() + 1e-10)

    # ---- losses ---------------------------------------------------------------------------
    def ev_ppo_loss(self, i):
        V, lp = self.evaluate(i)
        ratios = torch.exp(lp - self.curr_log_probs[i])
        surr1 = ratios * self.A_k[i]
        surr2 = torch.clamp(ratios, 1 - self.clip, 1 + self.clip) * self.A_k[i]
        actor_loss = (-torch.min(surr1, surr2)).mean()
        critic_loss = nn.functional.mse_loss(V, self.curr_rtgs[i])
        self.logger["actor_losses"].append(actor_loss.detach())
        return actor_loss, critic_loss

    def local_batch_loss(self, i):
        """Problem-API hook of the consensus optimizers: actor and critic share no parameters,
        so the sum's gradient is the pair of separate gradients the reference uses."""
        a, c = self.ev_ppo_loss(i)
        return a + c

    def update_graph(self):
        return

    def evaluate_metrics(self, at_end=False):
        return

    def avg_episode_reward(self) -> float:
        return float(np.mean(self.logger["batch_rews"])) if self.logger["batch_rews"] else float("nan")

    def _log_summary(self):
        now = time.time_ns()
        dt = (now - self.logger["delta_t"]) / 1e9
        self.logger["delta_t"] = now
        al = torch.stack(self.logger["actor_losses"]).mean().item() if self.logger["actor_losses"] else float("nan")
        print(flush=True)
        print(f"-------------------- Iteration #{self.logger['i_so_far']} --------------------", flush=True)
        print(f"Average Episodic Length: {np.mean(self.logger['batch_lens']):.2f}", flush=True)
        print(f"Average Episodic Return: {self.avg_episode_reward():.2f}", flush=True)
        print(f"Average Loss: {al:.5f}", flush=True)
        print(f"Timesteps So Far: {self.logger['t_so_far']}", flush=True)
        print(f"Iteration took: {dt:.2f} secs", flush=True)
        print("------------------------------------------------------", flush=True)
        self.logger["actor_losses"] = []
