"""K-GT — gradient tracking with local steps (Liu, Lin, Koloskova, Stich, *Decentralized Gradient Tracking with Local
Steps*, 2023), and local DSGD (Koloskova, Loizou, Boreiri, Jaggi, Stich, ICML 2020) with ``correction: false``.  No
counterpart in the reference.

Every round takes ``local_steps`` (K) gradient steps and communicates once.  Local DSGD carries DSGD's bias on
heterogeneous data, and the local steps make it worse; K-GT adds a correction row ``c_i`` that tracks the gap between
the node's mean direction and the network's, so the fixed point is the minimiser of ``sum_i f_i``.  With a constant
step ``alpha`` (the paper's inner step; its outer step is fixed at 1), round k of node i is, in this engine's
mix-first order,

    mix:   theta_i <- sum_j W_ij theta_j^pub                    (own term included)
           c_i     <- c_i + sum_j W_ij y_j^pub - y_i^pub        (correction only)
    for p = 0 .. K-1:   g_i = grad loss_i(theta_i)              (one minibatch draw per step)
           u_i = g_i + c_i  (g_i without correction);  theta_i <- theta_i - alpha u_i
           d_i <- u_i (p = 0) or d_i + u_i
    publish theta_i and y_i = d_i / K                           (y only with correction)

Everything starts at zero (c, and the published y of round 0), so round 0 is a local-DSGD round and no extra
gradient is drawn; the paper may start c from a first gradient.  Since W is doubly stochastic, ``sum_i c_i = 0`` every
round.  With K = 1 the iterates are DSGT's with ``init_grads: false``: ``g_i + c_i`` is DSGT's tracker and the mixed
rows are DSGT's.  Local DSGD with K = 1 is DSGD with ``mu: 0``, bitwise.

Between rounds theta is the model after the local steps and before the gossip (it equals the published row, as for
DSGD).  The checkpoint carries ``c`` and ``y``; ``d`` lives within a round.  Only the synchronous (Jacobi) order on
undirected graphs exists; changing graphs and link drops are allowed, as for DSGT.
"""
from __future__ import annotations

import numbers

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


def check_local_steps(v) -> int:
    """``local_steps`` must be an integer >= 1 (a bool or a float is refused)."""
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or int(v) < 1:
        raise ValueError(f"kgt local_steps must be an integer >= 1 (got {v!r})")
    return int(v)


class KGT(ConsensusOptimizer):
    alg_name = "kgt"

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("kgt runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and hasattr(graph, "is_directed") and graph.is_directed():
            raise ValueError("kgt needs an undirected graph (a doubly stochastic Metropolis matrix)")
        self.alpha = float(conf["alpha"])
        if not self.alpha > 0.0:
            raise ValueError(f"kgt alpha must be > 0 (got {conf['alpha']!r})")
        self.local_steps = check_local_steps(conf["local_steps"])
        self.correction = bool(conf.get("correction", True))
        self.refresh_graph = bool(conf.get("update_graph", True))
        a = self.arena
        self.c = a.zeros() if self.correction else None
        self.y = a.zeros() if self.correction else None      # the published tracker of the last round
        self.d = a.zeros() if self.correction else None      # the round's direction sum (dead between rounds)
        self.STATE = ("c", "y") if self.correction else ()

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        with torch.no_grad():
            theta_all = pr.gather_rows(a.theta)
            y_all = pr.gather_rows(self.y) if self.correction else None
            ref.kgt_mix_(a.theta, self.c, theta_all, y_all, self.y, self._rows(topo, topo.W))
        for p in range(self.local_steps):
            pr.compute_grads()
            with torch.no_grad():
                y = ref.kgt_step_(a.theta, self.c, self.d, a.grad, self.alpha, p, self.local_steps)
        if self.correction:
            self.y.copy_(y)
