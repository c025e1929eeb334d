"""Centralized PPO baseline: one shared actor/critic controls every predator
(reference: RL/ppo.py:71-170 ``learn``, RL/network.py)."""
from __future__ import annotations

import math
import os
import time

import numpy as np
import torch
from torch import nn
from torch.optim import Adam

from .gae import check_gae_lambda, gae
from .simple_tag import SimpleTagEnv, heuristic_prey_action


class PPO:
    # gae_lambda: None keeps the Monte-Carlo advantages rtgs - V and the critic target rtgs; a float in [0, 1] makes
    # them GAE(lambda) advantages and lambda-returns (rl/gae.py), on both update backends.  A batch's samples are
    # rows ((ep * T + c) * E + e) * n_adv + i, so each episode is T cycles of E * n_adv (world, predator) columns.
    DEFAULTS = dict(timesteps_per_batch=4800, max_timesteps_per_episode=1600, n_updates_per_iteration=5,
                    lr=0.005, gamma=0.95, clip=0.2, render=False, render_every_i=10, save_freq=10, seed=None,
                    ID=0, out_dir="./trained", rollout_backend="torch", update_backend="torch", gae_lambda=None)

    def __init__(self, policy_class, env: SimpleTagEnv, **hyperparameters):
        for k, v in {**self.DEFAULTS, **hyperparameters}.items():
            if k not in self.DEFAULTS:
                raise TypeError(f"unknown PPO hyper-parameter {k!r}")
            setattr(self, k, v)
        self.gae_lambda = check_gae_lambda(self.gae_lambda)
        if self.seed is not None:
            torch.manual_seed(self.seed)
        self.env = env
        self.obs_dim = env.observation_spaces["adversary_0"].shape[0]
        self.act_dim = env.action_spaces["adversary_0"].shape[0]
        self.actor = policy_class([self.obs_dim, 64, 64, 64, self.act_dim]).to(env.device)
        self.critic = policy_class([self.obs_dim, 64, 64, 64, 1]).to(env.device)
        self.actor_optim = Adam(self.actor.parameters(), lr=self.lr)
        self.critic_optim = Adam(self.critic.parameters(), lr=self.lr)
        self.cov_var = 0.5
        self.logger = {"delta_t": time.time_ns(), "t_so_far": 0, "i_so_far": 0, "batch_lens": [], "batch_rews": [],
                       "actor_losses": []}
        self.avg_ep_rews, self.timesteps = [], []
        if self.rollout_backend not in ("torch", "cuda"):
            raise ValueError(f"rollout_backend must be 'torch' or 'cuda', not {self.rollout_backend!r}")
        if self.rollout_backend == "cuda":
            from ..ops import tag_rollout
            tag_rollout.require(env, self.actor)
        self._rollout_key, self._rollout_index = None, 0
        if self.update_backend not in ("torch", "cuda"):
            raise ValueError(f"update_backend must be 'torch' or 'cuda', not {self.update_backend!r}")
        if self.update_backend == "cuda":
            from ..ops import ppo_update
            ppo_update.require(self.actor, self.critic)

    def _log_prob(self, mean, act):
        k = act.shape[-1]
        return -0.5 * ((act - mean) ** 2).sum(-1) / self.cov_var - 0.5 * k * math.log(2 * math.pi * self.cov_var)

    def get_action(self, obs):
        with torch.no_grad():
            mean = self.actor(obs)
            act = mean + math.sqrt(self.cov_var) * torch.randn_like(mean)
            return act, self._log_prob(mean, act)

    def evaluate(self, obs, acts):
        return self.critic(obs).squeeze(-1), self._log_prob(self.actor(obs), acts)

    def rollout(self):
        """One batch: ``(obs, acts, log_probs, rtgs, episode lengths)``, one row per (cycle, world, predator).  Under
        ``gae_lambda`` the per-cycle rewards of those rows and the episodes' cycle count are kept as ``self.rews`` and
        ``self.episode_T`` for the update."""
        if self.rollout_backend == "cuda":
            return self._rollout_cuda()
        env = self.env
        cycles = max(1, self.max_timesteps_per_episode // env.num_agents)
        obs_b, act_b, lp_b, rtg_b, rew_b, ep_ret, ep_len, t = [], [], [], [], [], [], [], 0
        while t < self.timesteps_per_batch:
            obs_adv, obs_good = env.reset()
            rews = []
            for c in range(cycles):
                flat = obs_adv.reshape(-1, self.obs_dim)
                a, lp = self.get_action(flat)
                acts = torch.zeros(env.E, env.A, 5, device=env.device, dtype=obs_adv.dtype)
                acts[:, : env.n_adv] = a.reshape(env.E, env.n_adv, 5)
                acts[:, env.n_adv:] = heuristic_prey_action(obs_good[:, 0], env.n_adv).unsqueeze(1)
                obs_b.append(flat); act_b.append(a); lp_b.append(lp)
                r_adv, _, done = env.step(acts)
                rews.append(r_adv)
                obs_adv, obs_good = env.observe()
                t += env.n_adv * env.E
                if done:
                    break
            R = torch.stack(rews)
            rtg, run = torch.zeros_like(R), torch.zeros_like(R[0])
            for s in range(R.shape[0] - 1, -1, -1):
                run = R[s] + self.gamma * run
                rtg[s] = run
            rtg_b.append(rtg.reshape(-1))
            rew_b.append(R)
            ep_ret.extend(R.sum(0).sum(-1).tolist()); ep_len.extend([R.shape[0] * env.num_agents] * env.E)
        self.logger["batch_rews"], self.logger["batch_lens"] = ep_ret, ep_len
        if self.gae_lambda is not None:
            lens = {r.shape[0] for r in rew_b}
            if len(lens) != 1:   # every episode runs min(cycles, max_cycles) cycles from a reset
                raise RuntimeError(f"GAE needs episodes of one length, got {sorted(lens)}")
            self.rews, self.episode_T = torch.cat([r.reshape(-1) for r in rew_b]), lens.pop()
        return torch.cat(obs_b), torch.cat(act_b), torch.cat(lp_b), torch.cat(rtg_b), ep_len

    def _rollout_cuda(self):
        """``rollout()`` as one kernel launch with the shared actor; samples come back in the torch path's
        [cycle, world, predator] order."""
        from ..ops import tag_rollout
        env = self.env
        T = min(max(1, self.max_timesteps_per_episode // env.num_agents), env.max_cycles)
        n_ep = max(1, -(-self.timesteps_per_batch // (env.n_adv * env.E * T)))
        if self._rollout_key is None:
            self._rollout_key = tag_rollout.draw_key()
        out = tag_rollout.rollout(env, self.actor, T=T, n_ep=n_ep, gamma=self.gamma, cov_var=self.cov_var,
                                  key=self._rollout_key, index=self._rollout_index, rews=self.gae_lambda is not None)
        self._rollout_index += 1
        flat = lambda x: x.transpose(0, 1).reshape(-1, *x.shape[2:])      # [N, R, ...] -> [R * N, ...]
        if self.gae_lambda is not None:
            self.rews, self.episode_T = flat(out["rews"]), T
        ep_len = [T * env.num_agents] * (n_ep * env.E)
        self.logger["batch_rews"], self.logger["batch_lens"] = out["ep_returns"].tolist(), ep_len
        return flat(out["obs"]), flat(out["acts"]), flat(out["log_probs"]), flat(out["rtgs"]), ep_len

    def learn(self, total_timesteps):
        print(f"Learning... Running {self.max_timesteps_per_episode} timesteps per episode, "
              f"{self.timesteps_per_batch} timesteps per batch for a total of {total_timesteps} timesteps")
        t_so_far = i_so_far = 0
        while t_so_far < total_timesteps:
            obs, acts, lps, rtgs, lens = self.rollout()
            t_so_far += int(np.sum(lens)); i_so_far += 1
            self.logger["t_so_far"], self.logger["i_so_far"] = t_so_far, i_so_far
            if self.update_backend == "cuda":
                self._update_cuda(obs, acts, lps, rtgs)
            else:
                self._update_torch(obs, acts, lps, rtgs)
            self.avg_ep_rews.append(float(np.mean(self.logger["batch_rews"])))
            self.timesteps.append(t_so_far)
            self._log_summary()
            if i_so_far % self.save_freq == 0:
                self.save()
            if self.render and i_so_far % self.render_every_i == 0:
                self.render_episode(i_so_far)

    def _advantages_torch(self, obs, acts, rtgs):
        """Normalised advantages and the critic target of one batch on the torch update path: ``rtgs - V`` and
        ``rtgs``, or under ``gae_lambda`` the GAE(lambda) advantages and lambda-returns."""
        with torch.no_grad():
            V, _ = self.evaluate(obs, acts)
        if self.gae_lambda is None:
            A = rtgs - V
        else:
            A, rtgs = gae(self.rews, V, self.gamma, self.gae_lambda, self.episode_T, self.env.E * self.env.n_adv)
        return (A - A.mean()) / (A.std() + 1e-10), rtgs

    def _update_torch(self, obs, acts, lps, rtgs):
        A, rtgs = self._advantages_torch(obs, acts, rtgs)
        for _ in range(self.n_updates_per_iteration):
            V, cur = self.evaluate(obs, acts)
            ratios = torch.exp(cur - lps)
            actor_loss = (-torch.min(ratios * A, torch.clamp(ratios, 1 - self.clip, 1 + self.clip) * A)).mean()
            critic_loss = nn.functional.mse_loss(V, rtgs)
            self.actor_optim.zero_grad(); actor_loss.backward(); self.actor_optim.step()
            self.critic_optim.zero_grad(); critic_loss.backward(); self.critic_optim.step()
            self.logger["actor_losses"].append(actor_loss.detach())

    def _update_cuda(self, obs, acts, lps, rtgs):
        """The same update with the fused kernels (ops/ppo_update.py): the batch is one node of the kernels' [N, R, ...]
        layout; each step's gradients land in p.grad and the two Adam steps run as on the torch path."""
        from ..ops import ppo_update
        obs, acts, lps, rtgs = obs.unsqueeze(0), acts.unsqueeze(0), lps.unsqueeze(0), rtgs.unsqueeze(0)
        if self.gae_lambda is None:
            A = ppo_update.advantages(self.critic, obs, rtgs)
        else:   # the critic's target becomes the lambda-return
            g = ppo_update.GAE(rews=self.rews.unsqueeze(0), gamma=self.gamma, lam=self.gae_lambda, T=self.episode_T,
                               E=self.env.E * self.env.n_adv)
            A, rtgs = ppo_update.advantages(self.critic, obs, rtgs, gae=g)
        params = list(self.actor.parameters()) + list(self.critic.parameters())
        for _ in range(self.n_updates_per_iteration):
            for p in params:
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
            losses = ppo_update.grads(self.actor, self.critic, obs, acts, lps, rtgs, A, self.clip, self.cov_var,
                                      [[p.grad for p in params]])
            self.actor_optim.step()
            self.critic_optim.step()
            self.logger["actor_losses"].append(losses[0, 0])

    def render_episode(self, i):
        """``render=True``: an animated GIF of one episode of the current policy every ``render_every_i`` iterations
        (the reference opens a pyglet window during rollouts, RL/ppo.py:197-199)."""
        from .eval_policy import rollout, save_rollout_gif
        os.makedirs(self.out_dir, exist_ok=True)
        _, _, traj = rollout(self.actor, self.env, record=True, backend=self.rollout_backend)
        return save_rollout_gif(self.env, traj, os.path.join(self.out_dir, f"render_{self.ID}_{i}.gif"))

    def save(self):
        os.makedirs(self.out_dir, exist_ok=True)
        torch.save(self.actor.state_dict(), os.path.join(self.out_dir, f"ppo_actor_tag_{self.ID}.pth"))
        torch.save(self.critic.state_dict(), os.path.join(self.out_dir, f"ppo_critic_tag_{self.ID}.pth"))
        np.save(os.path.join(self.out_dir, f"avg_ep_rews_{self.ID}.npy"), np.asarray(self.avg_ep_rews))
        np.save(os.path.join(self.out_dir, f"timesteps_{self.ID}.npy"), np.asarray(self.timesteps))

    def _log_summary(self):
        now = time.time_ns(); dt = (now - self.logger["delta_t"]) / 1e9; self.logger["delta_t"] = now
        al = torch.stack(self.logger["actor_losses"]).mean().item()
        print(f"\n-------------------- Iteration #{self.logger['i_so_far']} --------------------", flush=True)
        print(f"Average Episodic Length: {np.mean(self.logger['batch_lens']):.2f}", flush=True)
        print(f"Average Episodic Return: {np.mean(self.logger['batch_rews']):.2f}", flush=True)
        print(f"Average Loss: {al:.5f}\nTimesteps So Far: {self.logger['t_so_far']}\nIteration took: {dt:.2f} secs", flush=True)
        self.logger["actor_losses"] = []
