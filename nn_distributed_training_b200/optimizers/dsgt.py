"""DSGT — decentralized SGD with gradient tracking
(reference: optimizers/dsgt.py:7-115).

    init: y_i = g_i = grad loss_i(theta_i^0)           (if init_grads)
    theta_i^{k+1} = sum_j W_ij (theta_j^k - alpha y_j^k)
    g_i^{k+1}     = grad loss_i(theta_i^{k+1})
    y_i^{k+1}     = sum_j W_ij y_j^k + g_i^{k+1} - g_i^k

The reference's per-tensor ``norm().item()`` host syncs (:100,105, SURVEY Q16)
are dropped.  ``mixing_order: reference`` reproduces its sequential sweeps.

The distributed-PPO variants (rl/consensus_ppo.py) also run on the fused kernels:
a per-coordinate step ``alpha`` (a tensor [n_pad]) and ``own_tracker_step``
    theta_i^{k+1} = sum_j W_ij theta_j^k - alpha y_i^k
"""
from __future__ import annotations

from typing import Dict

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class DSGT(ConsensusOptimizer):
    alg_name = "dsgt"
    STATE = ("y", "g")

    def __init__(self, ddl_problem, device, conf):
        super().__init__(ddl_problem, device, conf)
        self.alpha = float(conf["alpha"])   # may be replaced by a per-coordinate tensor [n_pad]
        self.own_tracker_step = bool(conf.get("own_tracker_step", False))
        self.init_grads = bool(conf["init_grads"])
        self.refresh_graph = bool(conf.get("update_graph", True))
        self.y = self.arena.zeros()
        self.g = self.arena.zeros()
        self._initialised = False

    def _before_training(self):
        if self._initialised:
            return
        self._initialised = True
        if self.init_grads:
            self.pr.compute_grads()  # consumes one batch per node, like the reference (:33-46)
            self.y.copy_(self.arena.grad)
            self.g.copy_(self.arena.grad)

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        if self.mixing_order == "reference":
            W = torch.as_tensor(topo.W, dtype=a.dtype, device=self.device)
            with torch.no_grad():
                ref.dsgt_mix_sequential_(a.theta, self.y, W, topo.neighbors, self.alpha)
            for i in range(pr.N):  # gradient + tracker update interleaved per node (:78-103)
                self._grad_one(i)
                with torch.no_grad():
                    ref.dsgt_track_sequential_row_(i, self.y, W, topo.neighbors[i], a.grad[i], self.g[i])
                    self.g[i].copy_(a.grad[i])
            return
        w_rows = self._rows(topo, topo.W)
        with torch.no_grad():
            theta_all = pr.gather_rows(a.theta)
            y_all = pr.gather_rows(self.y)
            if self.own_tracker_step:   # RL variant: theta_i <- sum_j W_ij theta_j - alpha y_i
                a.theta.copy_(ref.dsgd_mix(theta_all, w_rows) - self.alpha * self.y)
            else:
                a.theta.copy_(ref.dsgt_mix(theta_all, y_all, w_rows, self.alpha))
        pr.compute_grads()
        with torch.no_grad():
            self.y.copy_(ref.dsgt_track(y_all, w_rows, a.grad, self.g))
            self.g.copy_(a.grad)

    def _grad_one(self, i: int):
        pr = self.pr
        inner = getattr(pr, "inner", pr)
        loss = inner.local_batch_loss(i)
        grads = torch.autograd.grad(loss, list(pr.models[i].parameters()))
        pr.arena.set_row_from_grads(i, grads)

    # ``initialised`` is saved under another name than its attribute, and ``alpha`` may be a per-coordinate row
    def state_dict(self) -> Dict:
        sd = super().state_dict()
        sd.update(initialised=self._initialised,
                  alpha=self.alpha.detach().cpu().clone() if torch.is_tensor(self.alpha) else float(self.alpha))
        return sd

    def load_state_dict(self, sd: Dict):
        super().load_state_dict(sd)
        self._initialised = bool(sd["initialised"])
        if "alpha" in sd:
            self.alpha = sd["alpha"].to(self.device) if torch.is_tensor(sd["alpha"]) else float(sd["alpha"])
