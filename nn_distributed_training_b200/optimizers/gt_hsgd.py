"""GT-HSGD — gradient tracking with a hybrid variance-reduced estimator (Xin, Khan, Kar, *A Hybrid Variance-Reduced
Method for Decentralized Stochastic Non-Convex Optimization*, ICML 2021).  No counterpart in the reference.

Gradient tracking (DSGT) removes the bias that heterogeneous data causes, but not the minibatch noise: at a constant
step its iterates settle at a noise floor set by ``alpha sigma^2``.  GT-HSGD tracks a STORM-type estimator ``v`` instead
of the raw gradient.  It needs no full gradients and no large checkpoint batches, only one minibatch per round, on
which the gradient is taken twice: at the new iterate and at the previous one.  Round k of node i, with
``omb = 1 - beta`` computed once in float64 and rounded once to the arena dtype:

    theta_i <- sum_j W_ij (theta_j - alpha y_j)                  (DSGT's mix)
    g_i  = grad loss_i(theta_i;      xi_k)                       (draw k)
    gp_i = grad loss_i(theta_prev_i; xi_k)                       (the same draw, at the previous iterate)
    v_i' = g_i                         in round 0
         = g_i + omb (v_i - gp_i)      otherwise
    y_i  <- sum_j W_ij y_j + v_i' - v_i;   v_i <- v_i';   theta_prev_i <- theta_i

The state starts at ``y = 0``, ``v = 0`` and ``theta_prev = theta^0``; no initial gradient is drawn (as for K-GT and
DeTAG), so round 0 is a DSGT round with ``init_grads: false``.

Two deviations from the paper, both deliberate:

* The tracker correction ``v' - v`` sits outside W, as in this repository's DSGT (the reference's form); the paper
  puts it inside the mix.  Both keep ``sum_i y_i = sum_i v_i`` every round for a doubly stochastic W.
* ``v^0`` is one minibatch gradient, not the gradient of a larger first batch of size ``b0``.

With these choices ``beta = 1`` is DSGT with ``init_grads: false`` bit for bit, since ``g + 0 (finite) = g``.

The tracking invariant holds for any doubly stochastic W, so changing graphs and link drops are allowed, as for DSGT.
Directed graphs, ``mixing_order: reference`` and Byzantine attackers are refused, and so is a problem driven through
the reference's API (``ReferenceProblemAdapter``, e.g. the PPO problem): its ``local_batch_loss`` draws a minibatch
internally and cannot evaluate it again at a second point.  The checkpoint carries ``y``, ``v`` and ``theta_prev``.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .base import ConsensusOptimizer, ReferenceProblemAdapter
from ..ops import consensus_ref as ref


def check_beta(v) -> float:
    """``beta`` must be finite and in (0, 1]."""
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not (math.isfinite(float(v)) and 0.0 < float(v) <= 1.0):
        raise ValueError(f"gt_hsgd beta must be finite and in (0, 1] (got {v!r})")
    return float(v)


class GTHSGD(ConsensusOptimizer):
    alg_name = "gt_hsgd"
    STATE = ("y", "v", "theta_prev")

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("gt_hsgd runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        if isinstance(self.pr, ReferenceProblemAdapter):
            raise ValueError("gt_hsgd needs two gradients on the same minibatch, and a problem driven through the "
                             "reference API (local_batch_loss, e.g. the PPO problem) draws its batch internally and "
                             "cannot evaluate it at a second point")
        if self.pr.graph is not None and self.pr.graph.is_directed():
            raise ValueError("gt_hsgd needs an undirected graph (a doubly stochastic Metropolis matrix)")
        if conf.get("byzantine") is not None:
            raise ValueError("gt_hsgd does not model Byzantine attackers (clipped_gossip and bridge do)")
        self.alpha = float(conf["alpha"])
        if not (math.isfinite(self.alpha) and self.alpha > 0.0):
            raise ValueError(f"gt_hsgd alpha must be finite and > 0 (got {conf['alpha']!r})")
        self.beta = check_beta(conf["beta"])
        a = self.arena
        npdt = np.float32 if a.dtype == torch.float32 else np.float64
        self.omb = float(npdt(1.0 - self.beta))    # 1 - beta in float64, rounded once to the arena dtype
        self.refresh_graph = bool(conf.get("update_graph", True))
        self.y = a.zeros()
        self.v = a.zeros()
        self.theta_prev = a.theta.detach().clone()
        self.grad_prev = a.zeros()                  # the gradient at theta_prev (scratch of the PyTorch path)
        if self.pr.fused is not None:               # the forward/backward kernels' second, prev-point op
            self.pr.fused.enable_prev_point(self.theta_prev)

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        w_rows = self._rows(topo, topo.W)
        with torch.no_grad():
            y_all = pr.gather_rows(self.y)
            a.theta.copy_(ref.dsgt_mix(pr.gather_rows(a.theta), y_all, w_rows, self.alpha))
        pr.compute_grads_pair(self.theta_prev, self.grad_prev)
        with torch.no_grad():
            ref.hsgd_track_(self.y, self.v, self.theta_prev, y_all, w_rows, a.grad, self.grad_prev, a.theta, self.omb,
                            first=k == 0)
