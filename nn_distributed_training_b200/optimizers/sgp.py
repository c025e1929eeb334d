"""SGP — Stochastic Gradient Push (Assran, Loizou, Ballas, Rabbat, ICML 2019): decentralized SGD on push-sum gossip
(Kempe, Dobra, Gehrke 2003; subgradient-push, Nedić & Olshevsky 2015).  No counterpart in the reference.

Push-sum needs only a column-stochastic mixing matrix, which every node sets from its own out-degree,
``A_ij = 1 / (d_out(j) + 1)`` for ``j -> i`` and ``j = i`` (``Topology.push_weights``).  So SGP runs on directed graphs
(an edge ``u -> v`` of an ``nx.DiGraph``: v reads u's row) and on graphs that change during a run, with no
Metropolis rebuild.  Each node keeps a numerator row ``x`` and a float64 push-sum weight ``w`` (1 at the start).  With
DSGD's step schedule ``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})``, round k of node i is

    mix:   x_i <- sum_{j in in_k(i) + i} A_ij x_j^pub     w_i <- sum A_ij w_j^pub     theta_i <- x_i / w_i
    step:  x_i <- x_i - alpha_k grad loss_i(theta_i);  theta_i <- x_i / w_i;  publish (x_i, w_i)

State between rounds: ``theta = x / w`` (the de-biased model that evaluation, checkpoints and the metrics see), ``x``
and ``w`` are the published row.  On a doubly stochastic graph (the cycle, regular directed graphs) ``w`` stays 1 up
to rounding and SGP is DSGD.  Only the synchronous (Jacobi) order exists.
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class SGP(ConsensusOptimizer):
    alg_name = "sgp"
    STATE = ("x", "w")
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("sgp runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        g = getattr(self.pr, "graph", None)
        if pconf.get("fault_injection") and g is not None and g.is_directed():
            raise ValueError("sgp: link-drop fault_injection drops undirected edges and does not apply to a directed graph")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        a = self.arena
        self.x = a.theta.detach().clone()
        self.w = torch.ones(a.L, dtype=torch.float64, device=self.device)

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            x_all = pr.gather_rows(self.x)
            w_all = pr.gather_rows(self.w.view(-1, 1)).view(-1)
            ref.sgp_mix_(self.x, self.w, a.theta, x_all, w_all, self._rows(topo, topo.push_weights))
        pr.compute_grads()
        with torch.no_grad():
            ref.sgp_step_(self.x, self.w, a.theta, a.grad, self.alph)
