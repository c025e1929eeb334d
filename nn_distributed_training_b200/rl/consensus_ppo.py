"""DiNNO / DSGD / DSGT applied to the distributed PPO problem
(reference: RL/dist_rl/dinnoPPO.py:6-269, dsgdPPO.py:7-165, dsgtPPO.py:7-254).

The three classes are thin loops — rollout, advantages, consensus round(s), agreement metric,
periodic save — around the *generic* arena optimizers; the reference instead re-implements each
algorithm a second time for the actor/critic pair (with a list-aliasing bug in DSGD's critic
update, SURVEY Q18, which cannot occur here because a node's variable is one flat row).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from ..optimizers import DiNNO, DSGD, DSGT


def agreement(problem) -> np.ndarray:
    """Distance of each node's L2-normalised [actor||critic] vector to the network mean
    (RL/dist_rl/dinnoPPO.py:195-223)."""
    with torch.no_grad():
        rows = []
        for i in range(problem.N):
            a = torch.nn.utils.parameters_to_vector(problem.models[i].actor.parameters())
            c = torch.nn.utils.parameters_to_vector(problem.models[i].critic.parameters())
            rows.append(torch.cat([a, c]))
        th = torch.nn.functional.normalize(torch.stack(rows), dim=1)
        return torch.cdist(th, th.mean(0, keepdim=True)).reshape(-1).cpu().numpy()


def schedule_horizon(conf, problem, oits: int, rounds_per_iteration: int) -> int:
    """Rounds a trainer can run: every batch collects at least ``timesteps_per_batch`` steps (on both rollout paths),
    so ``train()`` stops after ``ceil(max_rl_timesteps / timesteps_per_batch)`` iterations at the latest, or at
    ``outer_iterations``.  At most ``oits``, the inner optimizer's round count."""
    its = min(int(conf.get("outer_iterations", 10 ** 12)),
              -(-int(conf["max_rl_timesteps"]) // int(problem.timesteps_per_batch)))
    return max(1, min(int(oits), its * int(rounds_per_iteration)))


class _ConsensusPPO:
    """``consensus_backend`` (conf): ``torch`` (default) runs each round as PyTorch ops from Python; ``fused`` runs an
    iteration's rounds on the sm_90a consensus kernels (ops/csrc/consensus.cu), replayed from one CUDA graph when the
    gradient step is the update kernels (update_backend "cuda") and eagerly around per-node autograd otherwise."""
    alg = "base"

    def __init__(self, ddl_problem, device, conf):
        self.pr, self.conf, self.device = ddl_problem, conf, torch.device(device)
        self.out_dir = conf.get("out_dir", "./trained")
        backend = conf.get("consensus_backend", "torch")
        if backend not in ("torch", "fused"):
            raise ValueError(f"consensus_backend must be 'torch' or 'fused', not {backend!r}")
        self.inner = self._make_inner()
        self.fused = backend == "fused"
        if self.fused:
            self.inner._use_engine()          # raises ValueError naming what the fused kernels cannot run
            self.inner.horizon = schedule_horizon(self.conf, self.pr, self.inner.oits, self.rounds_per_iteration())
            if self.pr.batched_grads is not None:
                self.pr.use_fixed_batch(self.steps_per_iteration())
            self._batch_version = None
        self.avg_ep_rews, self.timesteps, self.agreements = [], [], []

    def _make_inner(self):
        raise NotImplementedError

    def rounds_per_iteration(self) -> int:
        """Consensus rounds of one iteration."""
        return self.pr.n_updates_per_iteration

    def steps_per_iteration(self) -> int:
        """Gradient steps (``compute_grads`` calls) of one iteration."""
        return self.pr.n_updates_per_iteration

    def _consensus(self, k):
        if self.fused:
            return self._fused_rounds()
        for _ in range(self.rounds_per_iteration()):
            self.inner._round(k)

    def _fused_rounds(self):
        """The iteration's rounds on the fused kernels: ``inner.run_rounds``, the same rounds and schedule values as
        ``_round(k)`` on the torch path."""
        pr, inner = self.pr, self.inner
        if inner.alg_name == "dsgt":
            # the torch trainer never runs _before_training, so init_grads is not honoured there and y = g = 0 at the
            # first round; marking the tracker initialised keeps the engine from starting a dsgt_init of its own (after
            # a caller's _before_training the engine takes the optimizer's y and g, as it always does)
            inner._initialised = True
        prog = getattr(inner, "_program", None)
        if prog is not None and pr.batch_version != self._batch_version:
            prog.drop_graphs()               # the batch buffers moved (R changed): recapture against the new ones
        self._batch_version = pr.batch_version
        if pr.capturable_grads:
            pr.begin_steps()
        inner.run_rounds(self.rounds_per_iteration())
        if pr.capturable_grads:
            pr.end_steps()

    def agreement(self) -> np.ndarray:
        """``agreement(problem)`` of the current parameters; on the fused path the consensus-metric kernel's distance to
        the mean on the published rows (fp64 accumulation; the arena padding is zero), in the parameters' dtype."""
        if not self.fused:
            return agreement(self.pr)
        _, mean = self.inner._program.eng.consensus_metric(self.inner.k)
        return mean.reshape(-1).to(self.inner.arena.dtype).numpy()

    def train(self, profiler=None):
        k = 0
        while self.pr.logger["t_so_far"] < self.conf["max_rl_timesteps"] and k < self.conf.get("outer_iterations", 10 ** 12):
            self.pr.split_rollout_marl()
            self.pr.update_advantage()
            self._consensus(k)
            self.pr.check_update()
            self.avg_ep_rews.append(self.pr.avg_episode_reward())
            self.timesteps.append(self.pr.logger["t_so_far"])
            self.agreements.append(self.agreement())
            self.pr._log_summary()
            if profiler is not None:
                profiler.step()
            if k % self.pr.save_freq == 0 and self.conf.get("writeout", True):
                self.save(k)
            if getattr(self.pr, "render", False) and k % max(int(self.pr.render_every_i), 1) == 0:
                self.render_episode(k)
            k += 1
        return

    def render_episode(self, k):
        """Animated GIF of one episode with every predator running its own current actor (reference:
        RL/dist_rl/vids/*.mp4, rendered from the pyglet window)."""
        from .eval_policy import rollout, save_rollout_gif
        os.makedirs(self.out_dir, exist_ok=True)
        actors = [self.pr.models[i].actor for i in range(self.pr.N)]
        _, _, traj = rollout(actors, self.pr.env, record=True, backend=getattr(self.pr, "rollout_backend", "torch"))
        return save_rollout_gif(self.pr.env, traj, os.path.join(self.out_dir, f"{self.alg}_{self.conf.get('ID', 0)}_{k}.gif"))

    def save(self, k):
        os.makedirs(self.out_dir, exist_ok=True)
        ID, alg = self.conf.get("ID", 0), self.alg
        torch.save({f"actor{i}": self.pr.models[i].actor.state_dict() for i in range(self.pr.N)},
                   os.path.join(self.out_dir, f"ppo_actors_tag_{alg}_{ID}_{k}.pth"))
        torch.save({f"critic{i}": self.pr.models[i].critic.state_dict() for i in range(self.pr.N)},
                   os.path.join(self.out_dir, f"ppo_critics_tag_{alg}_{ID}_{k}.pth"))
        np.save(os.path.join(self.out_dir, f"avg_ep_rews_{alg}_{ID}.npy"), np.asarray(self.avg_ep_rews))
        np.save(os.path.join(self.out_dir, f"timesteps_{alg}_{ID}.npy"), np.asarray(self.timesteps))
        ag = np.asarray(self.agreements)
        np.savez(os.path.join(self.out_dir, f"agreements_{alg}_{ID}"),
                 **{f"agree_{i}": ag[:, i] for i in range(ag.shape[1])})


class DiNNOPPO(_ConsensusPPO):
    """conf: rho_init, rho_scaling, primal_lr_start/finish, lr_decay_type, persistant_primal_opt,
    primal_iterations, max_rl_timesteps, outer_iterations, ID (train_cadmm_multi.py:47-58)."""
    alg = "dinno"

    def _make_inner(self):
        c = dict(self.conf)
        c.setdefault("alg_name", "dinno")
        c.setdefault("primal_optimizer", "adam")
        c.setdefault("consensus_backend", "torch")
        return DiNNO(self.pr, self.device, c)

    def rounds_per_iteration(self) -> int:
        return 1

    def steps_per_iteration(self) -> int:
        return self.inner.pits


class DSGDPPO(_ConsensusPPO):
    """conf: alpha0, mu, max_rl_timesteps, ID; ``n_updates_per_iteration`` mix+step passes per rollout."""
    alg = "dsgd"

    def _make_inner(self):
        c = dict(self.conf)
        c.setdefault("alg_name", "dsgd")
        c.setdefault("outer_iterations", 10 ** 12)
        c.setdefault("consensus_backend", "torch")
        return DSGD(self.pr, self.device, c)


class DSGTPPO(_ConsensusPPO):
    """conf: alpha_actor, alpha_critic (per-slot step sizes), init_grads, max_rl_timesteps, ID.
    ``own_tracker_step`` reproduces the reference's theta_i <- sum_j W_ij theta_j - alpha y_i
    (RL/dist_rl/dsgtPPO.py:106-114) instead of the supervised form."""
    alg = "dsgt"

    def _make_inner(self):
        c = dict(self.conf)
        c.setdefault("alg_name", "dsgt")
        c.setdefault("outer_iterations", 10 ** 12)
        c.setdefault("init_grads", False)
        c.setdefault("consensus_backend", "torch")
        c.setdefault("own_tracker_step", True)
        c["alpha"] = float(c.get("alpha", c.get("alpha_actor", 1e-3)))
        inner = DSGT(self.pr, self.device, c)
        if "alpha_actor" in c and "alpha_critic" in c:
            alpha = torch.zeros(inner.arena.n_pad, dtype=inner.arena.dtype, device=self.device)
            for s in inner.arena.layout.slots:
                alpha[s.offset: s.offset + s.numel] = c["alpha_actor"] if s.name.startswith("actor") else c["alpha_critic"]
            inner.alpha = alpha
        return inner
