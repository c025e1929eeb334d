"""BRIDGE — Byzantine-resilient decentralized gradient descent by coordinate-wise screening (Fang, Yang, Bajwa, *BRIDGE:
Byzantine-resilient decentralized gradient descent*, IEEE TSIPN 2022): the trimmed mean (BRIDGE-T) and the median
(BRIDGE-M).  No counterpart in the reference.

DSGD's step schedule (``alpha0``, ``mu``) and single published channel.  Round k of node i, in this engine's mix-first
order (``v_j = theta_j^pub``, the row neighbor j published at the end of round k-1), element by element:

    trimmed_mean (b):  sort the deg neighbor values; keep sorted positions [b, deg - b)  (none when deg <= 2b)
                       y = (theta_i + the kept values, summed in ascending order) / (1 + max(0, deg - 2b))
    median:            y = median of {theta_i} U {v_j}; of an even count 0.5 (lower + upper middle value)
    step:              theta_i <- y - alpha_k grad loss_i(y); publish theta_i (or the attack row)

The sum and the even-count average are taken in fp64 and rounded once to the row dtype, so the result does not depend
on the order of the neighbor table.  The own term is always the node's own theta_i, never the row it published (which
matters for a Byzantine node).  The paper takes the gradient at the pre-screen iterate; here it is taken at the screened
row, like every DSGD-family optimizer in this project.  Uniform weights over the kept values replace Metropolis weights,
so ``trimmed_mean`` with ``b: 0`` is the unweighted mean of the node and its neighbors, not DSGD.  A node with
``deg <= 2b`` keeps its own row that round (link drops and changing graphs are allowed, so this is not refused).

Byzantine nodes (``byzantine: {nodes, attack, scale, z}``) publish ClippedGossip's attack rows (``sign_flip``,
``alie``); those rows are optimizer state, carried by the checkpoint.  Only the synchronous (Jacobi) order on undirected
graphs exists.  The fused mix holds the neighbor values in registers, for at most 16 neighbors per node.
"""
from __future__ import annotations

import numbers

import torch

from .base import ConsensusOptimizer
from .clipped_gossip import setup_attackers
from ..ops import consensus_ref as ref


class Bridge(ConsensusOptimizer):
    alg_name = "bridge"
    STATE = ("pub",)
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("bridge runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and hasattr(graph, "is_directed") and graph.is_directed():
            raise ValueError("bridge needs an undirected graph (every neighbor reads the node's published row)")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.alph = self.alph0
        self.screen = conf["screen"]
        if self.screen not in ref.BRIDGE_SCREENS:
            raise ValueError(f"bridge screen must be one of {'|'.join(ref.BRIDGE_SCREENS)} (got {self.screen!r})")
        b = conf.get("b", 0) if self.screen == "trimmed_mean" else 0
        if isinstance(b, bool) or not isinstance(b, numbers.Integral) or b < 0:
            raise ValueError(f"bridge b must be an integer >= 0 (got {b!r})")
        self.b = int(b)
        self.refresh_graph = bool(conf.get("update_graph", True))
        setup_attackers(self, conf.get("byzantine"))
        self.pub = self.arena.theta.detach().clone()      # the rows the local nodes published last

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``), DSGD's schedule."""
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
        lo = pr.placement.lo
        with torch.no_grad():
            pub_all = pr.gather_rows(self.pub)
            ref.bridge_mix_(a.theta, pub_all, topo.neighbors_noself, lo, self.screen, self.b)
        pr.compute_grads()
        with torch.no_grad():
            ref.dsgd_step_(a.theta, a.grad, self.alph)
            ref.cg_publish_(self.pub, a.theta, pub_all, self.attack, topo.neighbors_noself, set(self.byzantine), lo,
                            self.scale, self.z)
