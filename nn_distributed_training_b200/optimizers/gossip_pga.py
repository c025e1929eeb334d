"""Gossip-PGA — gossip SGD with a periodic global average (Chen, Yuan, Zhang, Pan, Xu, Yin, *Accelerating Gossip SGD
with Periodic Global Averaging*, ICML 2021), and local SGD (Stich, ICLR 2019) with ``gossip: false``.  No counterpart
in the reference.

DSGD's round (mix, gradient at the mixed point, step) with DSGD's step schedule; every ``period``-th round replaces the
gossip mix with the exact network mean.  Round k of node i:

    alpha_k  = alpha_{k-1} (1 - mu alpha_{k-1})
    theta~_i = (1/N) sum_j theta_j^k              global round: k mod period == period - 1 (every node, any graph)
             = sum_{j in N_i + i} W_ij theta_j^k  gossip round, gossip: true (DSGD's Metropolis mix)
             = theta_i^k                          gossip round, gossip: false (local SGD: nothing is pulled)
    theta_i^{k+1} = theta~_i - alpha_k grad loss_i(theta~_i)

Index choice: the paper averages the output of step k when (k + 1) mod H == 0.  Under this repository's mix-then-step
order that average is the mix of round k + 1, so round k is global when k mod period == period - 1.  Two exact
equivalences follow: ``period > outer_iterations`` never averages and is DSGD, and ``period == 1`` averages every round
and is DSGD on the complete graph in sum mode (synchronous parallel SGD).

The global mean is accumulated in float64 (ops/consensus_ref.py: pga_mean_; the fused kernels reduce fp64 partial sums,
across GPUs with one NVLS reduction).  The state is DSGD's: the checkpoint carries ``alph`` and nothing else, and the
fused kernels derive the period phase from the device round counter.  Changing graphs and link drops are allowed and
affect gossip rounds only; directed graphs, ``mixing_order: reference`` and Byzantine attackers are refused.
"""
from __future__ import annotations

import math
import numbers

import networkx as nx
import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


def check_period(v, alg: str = "gossip_pga") -> int:
    """``period`` must be an integer >= 1 (a bool or a float is refused)."""
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or int(v) < 1:
        raise ValueError(f"{alg} period must be an integer >= 1 (got {v!r})")
    return int(v)


class GossipPGA(ConsensusOptimizer):
    alg_name = "gossip_pga"
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError(f"{self.alg_name} runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and graph.is_directed():
            raise ValueError(f"{self.alg_name} needs an undirected graph (a doubly stochastic Metropolis matrix)")
        if conf.get("byzantine") is not None:
            raise ValueError(f"{self.alg_name} does not model Byzantine attackers (clipped_gossip and bridge do)")
        self.alph0 = float(conf["alpha0"])
        if not (math.isfinite(self.alph0) and self.alph0 >= 0.0):
            raise ValueError(f"{self.alg_name} alpha0 must be finite and >= 0 (got {conf['alpha0']!r})")
        self.mu = float(conf.get("mu", 0.0))
        self.period = check_period(conf["period"], self.alg_name)
        self.gossip = conf.get("gossip", True)
        if not isinstance(self.gossip, bool):
            raise ValueError(f"{self.alg_name} gossip must be true or false (got {self.gossip!r})")
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``), DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def is_global(self, k: int) -> bool:
        return k % self.period == self.period - 1

    def edgeless_graph(self):
        """The base graph of local SGD on the fused kernels: the problem's nodes and no edge (no pointer rows, no
        neighbor waits)."""
        return nx.empty_graph(self.pr.N)

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:      # every round, so a link-drop sequence is the one the fused plan draws
            pr.update_graph()
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            if self.is_global(k):
                ref.pga_mean_(a.theta, pr.gather_rows(a.theta))
            elif self.gossip:
                topo = pr.topology()
                a.theta.copy_(ref.dsgd_mix(pr.gather_rows(a.theta), self._rows(topo, topo.W)))
        pr.compute_grads()
        with torch.no_grad():
            ref.dsgd_step_(a.theta, a.grad, self.alph)
