"""DiNNO — consensus ADMM with an inexact primal step
(reference: optimizers/dinno.py:6-130; equations SURVEY Appendix D).

Per round k (Jacobi — a snapshot theta^k of every node is taken first):
    rho_k   = rho_{k-1} * rho_scaling                       (scaled before first use, Q4)
    dual_i += rho_k * sum_j (theta_i^k - theta_j^k)
    theta_i <- `primal_iterations` optimizer steps on
               loss_i(theta) + theta.dual_i + rho_k sum_j |theta - (theta_i^k+theta_j^k)/2|^2
The quadratic term is never materialised: with delta_i = sum_j (theta_j^k - theta_i^k)
its gradient is ``2 rho d_i (theta - theta_i^k) - rho delta_i``, so a primal step is
one elementwise kernel over the arena row (ops/csrc/consensus.cu: dinno_update).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


def primal_lr_table(conf) -> np.ndarray:
    """Per-round primal learning rates: constant | linear | log
    (optimizers/dinno.py:17-34), computed in float64."""
    n = int(conf["outer_iterations"])
    kind = conf["lr_decay_type"]
    a = float(conf["primal_lr_start"])
    if kind == "constant":
        return np.full(n, a)
    b = float(conf["primal_lr_finish"])
    if kind == "linear":
        return np.linspace(a, b, n)
    if kind == "log":
        return np.logspace(math.log10(a), math.log10(b), n)
    raise NameError("Unknow primal learning rate decay type.")


class DiNNO(ConsensusOptimizer):
    alg_name = "dinno"
    STATE = ("duals", "m", "v")
    SCALARS = ("rho", "t")

    def __init__(self, ddl_problem, device, conf):
        super().__init__(ddl_problem, device, conf)
        self.rho = float(conf["rho_init"])
        self.rho_scaling = float(conf["rho_scaling"])
        self._primal_lr = None   # materialised lazily: RL runs use outer_iterations ~ 1e7 with a constant rate
        self.pits = int(conf["primal_iterations"])
        self.opt_kind = conf["primal_optimizer"]
        if self.opt_kind not in ("adam", "sgd", "adamw"):
            raise NameError("DiNNO primal optimizer is unknown.")
        self.persistent = bool(conf["persistant_primal_opt"])
        # Q5: the reference's persistent optimizer keeps lr = primal_lr[0] forever;
        # opt into the schedule with `persistent_follows_schedule: true`.
        self.persistent_follows_schedule = bool(conf.get("persistent_follows_schedule", False))
        a = self.arena
        self.duals = a.zeros()
        self.delta = a.zeros()
        self.m = a.zeros() if self.opt_kind != "sgd" else None
        self.v = a.zeros() if self.opt_kind != "sgd" else None
        self.t = 0  # optimizer step count (persistent mode)

    def rho_at(self, k: int) -> float:
        """rho used in round k (rho_init * scaling^(k+1))."""
        return float(self.conf["rho_init"]) * self.rho_scaling ** (k + 1)

    @property
    def primal_lr(self):
        if self._primal_lr is None:
            self._primal_lr = primal_lr_table(self.conf)
        return self._primal_lr

    @primal_lr.setter
    def primal_lr(self, table):
        self._primal_lr = np.asarray(table, dtype=np.float64)

    def lr_at(self, k: int) -> float:
        if self.conf["lr_decay_type"] == "constant" and self._primal_lr is None:
            return float(self.conf["primal_lr_start"])
        if self.persistent and not self.persistent_follows_schedule:
            return float(self.primal_lr[0])
        return float(self.primal_lr[k])

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        theta_all = pr.gather_rows(a.theta).clone()  # snapshot theta^k of every node
        theta_k = a.theta.clone()
        self.rho *= self.rho_scaling
        pr.update_graph()
        topo = pr.topology()
        deg = self._deg(topo)
        ref.dinno_exchange_(theta_k, theta_all, self._rows(topo, topo.adj.astype(np.float64)),
                            deg, self.rho, self.duals, self.delta)
        lr = self.lr_at(k)
        if not self.persistent:
            self.t = 0
            if self.m is not None:
                self.m.zero_()
                self.v.zero_()
        for _ in range(self.pits):
            pr.compute_grads()
            g = ref.dinno_grad(a.theta, theta_k, a.grad, self.duals, self.delta, deg, self.rho)
            self.t += 1
            with torch.no_grad():
                ref.optimizer_step_(a.theta, g, self.opt_kind, lr, self.m, self.v, self.t)
