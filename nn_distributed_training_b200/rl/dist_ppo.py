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

from .gae import check_gae_lambda, gae
from .model import ActorCritic
from .simple_tag import SimpleTagEnv, heuristic_prey_action


BATCH_KEYS = ("obs", "acts", "log_probs", "rtgs")
GAE_KEYS = BATCH_KEYS + ("rews",)   # the batch under gae_lambda: the per-cycle rewards too


class DistPPOProblem:
    # defaults of the reference's _init_hyperparameters (:391-436) — set explicitly, no exec()
    # rollout_backend "cuda": each batch is one fused kernel launch (ops/tag_rollout.py) with its own Philox noise stream
    # update_backend "cuda": advantages and every node's gradients per primal step are fused kernels (ops/ppo_update.py);
    # a non-finite actor mean then raises from check_update(), which the trainers call at the end of every iteration,
    # and at the latest from the next update_advantage() -- not inside the primal step as on the torch path
    # gae_lambda: None keeps the Monte-Carlo advantages rtgs - V and the critic target rtgs; a float in [0, 1] makes
    # them GAE(lambda) advantages and lambda-returns (rl/gae.py), on both update backends
    DEFAULTS = dict(timesteps_per_batch=4800, max_timesteps_per_episode=1600, n_updates_per_iteration=5,
                    lr=0.005, gamma=0.95, clip=0.2, render=False, render_every_i=10, save_freq=10, seed=None,
                    rollout_backend="torch", update_backend="torch", gae_lambda=None)

    def __init__(self, base_actor, base_critic, graph, env: SimpleTagEnv, **hyperparameters):
        for k, v in {**self.DEFAULTS, **hyperparameters}.items():
            if k not in self.DEFAULTS:
                raise TypeError(f"unknown PPO hyper-parameter {k!r}")
            setattr(self, k, v)
        self.gae_lambda = check_gae_lambda(self.gae_lambda)
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
        if self.update_backend not in ("torch", "cuda"):
            raise ValueError(f"update_backend must be 'torch' or 'cuda', not {self.update_backend!r}")
        # batched gradient hook of ReferenceProblemAdapter.compute_grads (None: per-node autograd)
        self.batched_grads = None
        # fused consensus (use_fixed_batch): the batch lives in persistent buffers, so the gradient step can be replayed
        self.fixed_batch = False
        self.batch_version = 0
        if self.update_backend == "cuda":
            from ..ops import ppo_update
            ppo_update.require(self.actors, self.critics)
            self.batched_grads = self._cuda_grads
            self._nonfinite = torch.zeros(1, device=self.device, dtype=torch.int32)
            self._checked = True   # the flag holds nothing unchecked

    @property
    def capturable_grads(self) -> bool:
        """True when ``batched_grads`` reads only tensors at fixed addresses and has no per-call host side effects, so
        the consensus rounds around it can be captured in a CUDA graph and replayed (``ReferenceProblemAdapter``)."""
        return self.fixed_batch and self.batched_grads is not None

    @property
    def batch_keys(self):
        return BATCH_KEYS if self.gae_lambda is None else GAE_KEYS

    def use_fixed_batch(self, steps_per_iteration: int):
        """Fused-consensus mode of the trainers: from the next batch on, ``obs`` / ``acts`` / ``log_probs`` / ``rtgs``
        (and, under ``gae_lambda``, ``rews`` and the lambda-returns) and the advantages live in persistent
        ``[N, R, ...]`` buffers (reallocated, with ``batch_version`` bumped, only
        when R changes) and each primal step's ``[N, 2]`` losses go to row ``s`` of ``step_losses [steps_per_iteration,
        N, 2]``, s counted from ``begin_steps()``; ``end_steps()`` then logs them.  ``curr_*[i]`` / ``A_k[i]`` stay views of
        row i."""
        self.fixed_batch = True
        self._bufs = None
        self._loss_step = 0
        self._in_steps = False
        if self.update_backend == "cuda":
            p = next(self.models[0].parameters())
            self.step_losses = torch.zeros(int(steps_per_iteration), self.N, 2, device=p.device, dtype=p.dtype)

    def _into_buffers(self, out):
        b, keys = self._bufs, self.batch_keys
        if b is None or any(b[k].shape != out[k].shape or b[k].dtype != out[k].dtype for k in keys):
            b = self._bufs = {k: torch.empty(out[k].shape, dtype=out[k].dtype, device=out[k].device) for k in keys}
            b["adv"] = torch.empty(out["rtgs"].shape, dtype=out["rtgs"].dtype, device=out["rtgs"].device)
            if self.gae_lambda is not None:
                b["returns"] = torch.empty_like(b["adv"])
            self.batch_version += 1
        for k in keys:
            if out[k] is not b[k]:
                b[k].copy_(out[k])
        return b

    def begin_steps(self):
        """Fused consensus: the next primal step writes its losses into row 0 of ``step_losses``."""
        self._loss_step = 0
        self._in_steps = True

    def end_steps(self):
        """Fused consensus, after the steps of an iteration ran (replayed or eager): log their actor losses as the
        update path does and mark the non-finite flag unchecked for ``check_update()``."""
        self._in_steps = False
        if self.update_backend != "cuda":
            return
        vals = self.step_losses.clone()
        self.logger["actor_losses"].extend(vals[s, i, 0] for s in range(vals.shape[0]) for i in range(self.N))
        self._checked = False

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
        lp_b = [[] for _ in range(N)]; rtg_b = [[] for _ in range(N)]; rew_b = [[] for _ in range(N)]
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
                rew_b[i].append(R[:, :, i])
            ep_returns.extend(R.sum(0).sum(-1).tolist())            # joint predator return per world
            ep_lens.extend([R.shape[0] * env.num_agents] * env.E)
        flat = lambda xs: torch.cat([x.reshape(-1, *x.shape[2:]) if x.dim() > 2 else x.reshape(-1) for x in xs])
        self.curr_obs = {i: torch.cat(obs_b[i]) for i in range(N)}
        self.curr_acts = {i: torch.cat(act_b[i]) for i in range(N)}
        self.curr_log_probs = {i: torch.cat(lp_b[i]) for i in range(N)}
        self.curr_rtgs = {i: torch.cat([r.reshape(-1) for r in rtg_b[i]]) for i in range(N)}
        if self.gae_lambda is not None:
            self.curr_rews = {i: torch.cat([r.reshape(-1) for r in rew_b[i]]) for i in range(N)}
            lens = {r.shape[0] for r in rew_b[0]}
            if len(lens) != 1:   # every episode runs min(cycles, max_cycles) cycles from a reset
                raise RuntimeError(f"GAE needs episodes of one length, got {sorted(lens)}")
            self._episode_T = lens.pop()
        if self.update_backend == "cuda":
            self._stack_batch({k: torch.stack([getattr(self, "curr_" + k)[i] for i in range(N)])
                               for k in self.batch_keys})
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
        b, R = getattr(self, "_bufs", None), n_ep * T * env.E
        into = {k: b[k] for k in self.batch_keys} if self.fixed_batch and b is not None and b["rtgs"].shape == (N, R) \
            else None
        out = tag_rollout.rollout(env, self.actors, T=T, n_ep=n_ep, gamma=self.gamma, cov_var=self.cov_var,
                                  key=self._rollout_key, index=self._rollout_index, out=into,
                                  rews=self.gae_lambda is not None)
        self._rollout_index += 1
        self._episode_T = T
        self._stack_batch(out)
        ep_lens = [T * env.num_agents] * (n_ep * env.E)
        self.logger["batch_rews"] = out["ep_returns"].tolist()
        self.logger["batch_lens"] = ep_lens
        self.logger["t_so_far"] += int(np.sum(ep_lens))
        self.logger["i_so_far"] += 1

    def _stack_batch(self, out):
        """Keep the batch as ``[N, R, ...]`` tensors (the update kernels' layout); ``curr_*[i]`` are views of row i."""
        if self.fixed_batch:
            out = self._into_buffers(out)
        self._batch = {k: out[k] for k in self.batch_keys}
        self.curr_obs = {i: out["obs"][i] for i in range(self.N)}
        self.curr_acts = {i: out["acts"][i] for i in range(self.N)}
        self.curr_log_probs = {i: out["log_probs"][i] for i in range(self.N)}
        self.curr_rtgs = {i: out["rtgs"][i] for i in range(self.N)}
        if self.gae_lambda is not None:
            self.curr_rews = {i: out["rews"][i] for i in range(self.N)}

    def compute_rtgs(self, batch_rews):
        out = []
        for ep in reversed(batch_rews):
            d = 0.0
            for r in reversed(ep):
                d = r + d * self.gamma
                out.insert(0, d)
        return torch.tensor(out, dtype=torch.float)

    def update_advantage(self):
        """Per-node normalised advantages ``A_k`` of the critics at the start of the iteration, and the critic targets:
        ``rtgs - V`` and ``rtgs``, or under ``gae_lambda`` the GAE(lambda) advantages and lambda-returns of each
        episode of the batch (``curr_returns``)."""
        if self.update_backend == "cuda":
            from ..ops import ppo_update
            self.check_update()   # the previous iteration's steps, if the driver did not check them
            b, bufs = self._batch, self._bufs if self.fixed_batch else None
            out = bufs["adv"] if bufs is not None else None
            if self.gae_lambda is None:
                self._adv = ppo_update.advantages(self.critics, b["obs"], b["rtgs"], out=out)
            else:
                g = ppo_update.GAE(rews=b["rews"], gamma=self.gamma, lam=self.gae_lambda, T=self._episode_T,
                                   E=self.env.E, returns=bufs["returns"] if bufs is not None else None)
                self._adv, self._returns = ppo_update.advantages(self.critics, b["obs"], b["rtgs"], out=out, gae=g)
                self.curr_returns = {i: self._returns[i] for i in range(self.N)}
            self.A_k = {i: self._adv[i] for i in range(self.N)}
            return
        self.A_k = {}
        if self.gae_lambda is not None:
            self.curr_returns = {}
        with torch.no_grad():
            for i in range(self.N):
                V, _ = self.evaluate(i)
                if self.gae_lambda is None:
                    A = self.curr_rtgs[i] - V                         # ALG STEP 5
                else:
                    A, self.curr_returns[i] = gae(self.curr_rews[i], V, self.gamma, self.gae_lambda,
                                                  self._episode_T, self.env.E)
                self.A_k[i] = (A - A.mean()) / (A.std() + 1e-10)

    def critic_target(self, i):
        """Node i's critic target: the rewards-to-go, or the lambda-returns under ``gae_lambda``."""
        return self.curr_rtgs[i] if self.gae_lambda is None else self.curr_returns[i]

    # ---- losses ---------------------------------------------------------------------------
    def ev_ppo_loss(self, i):
        V, lp = self.evaluate(i)
        ratios = torch.exp(lp - self.curr_log_probs[i])
        surr1 = ratios * self.A_k[i]
        surr2 = torch.clamp(ratios, 1 - self.clip, 1 + self.clip) * self.A_k[i]
        actor_loss = (-torch.min(surr1, surr2)).mean()
        critic_loss = nn.functional.mse_loss(V, self.critic_target(i))
        self.logger["actor_losses"].append(actor_loss.detach())
        return actor_loss, critic_loss

    def local_batch_loss(self, i):
        """Problem-API hook of the consensus optimizers: actor and critic share no parameters,
        so the sum's gradient is the pair of separate gradients the reference uses."""
        a, c = self.ev_ppo_loss(i)
        return a + c

    def _cuda_grads(self, grad_out):
        """Every node's gradient of ``local_batch_loss`` at once (update_backend "cuda"): fills ``grad_out[i]`` (one
        tensor per parameter of models[i]) and returns the per-node losses ``[N, 2]`` without a host synchronisation."""
        from ..ops import ppo_update
        b = self._batch
        target = b["rtgs"] if self.gae_lambda is None else self._returns   # a persistent buffer under fixed_batch
        if self.fixed_batch:     # fused consensus: replayable, the trainer logs step_losses after the iteration
            slot = self._loss_step % self.step_losses.shape[0]
            self._loss_step += 1
            losses = ppo_update.grads(self.actors, self.critics, b["obs"], b["acts"], b["log_probs"], target,
                                      self._adv, self.clip, self.cov_var, grad_out, nonfinite=self._nonfinite,
                                      losses_out=self.step_losses[slot])
            self._checked = False
            if not self._in_steps:   # a step outside the trainer's iteration (DSGT's init_grads): logged as it runs
                self.logger["actor_losses"].extend(losses.clone()[:, 0])
            return losses
        losses = ppo_update.grads(self.actors, self.critics, b["obs"], b["acts"], b["log_probs"], target,
                                  self._adv, self.clip, self.cov_var, grad_out, nonfinite=self._nonfinite)
        self.logger["actor_losses"].extend(losses[i, 0] for i in range(self.N))
        self._checked = False
        return losses

    def check_update(self):
        """End of an iteration: under update_backend "cuda", raise if any actor mean of the primal steps since the last
        check was not finite (the torch path raises inside the step).  One host synchronisation, none if no step ran
        since the last check."""
        if self.update_backend != "cuda" or self._checked:
            return
        bad = int(self._nonfinite.item())
        self._nonfinite.zero_()
        self._checked = True
        if bad:
            raise NameError("actor returning something weird")

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
