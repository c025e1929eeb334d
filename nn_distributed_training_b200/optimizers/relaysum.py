"""RelaySum — exact averaging relayed over a spanning tree (Vogels, He, Koloskova, Karimireddy, Lin, Stich, Jaggi,
*RelaySum for Decentralized Deep Learning on Heterogeneous Data*, NeurIPS 2021).  No counterpart in the reference.

On a fixed undirected tree each node sends each neighbor a *different* message: its own model plus what its other
neighbors relayed to it.  After ``diam`` rounds every node averages all ``n`` models exactly, each one delayed by its
hop distance, so heterogeneous data biases nothing: there is no Metropolis weighting, no second channel and no tracker.
``N(i)`` is node i's neighbor list (``Topology.neighbors_noself[i]``), ``R_i^k = |{l : d(i, l) <= k}|`` (i included)
and ``alpha_k`` is DSGD's schedule.  Between rounds ``theta_i`` holds the half-step ``h_i`` (the initial parameters
before round 0), and node i has published one message ``m_{i->j}`` per neighbor (all zero before round 0).  Round k of
node i, in this engine's mix -> gradient -> step order:

    mix:   r_e <- m_{j_e -> i}          for each neighbor j_e, e = 0 .. deg_i - 1   (published at the end of round k-1)
           x_i <- h_i + (sum_e r_e - (R_i^k - 1) h_i) / n;   theta_i <- x_i
    fwd/bwd at x_i: g_i
    step:  h_i <- x_i - alpha_k g_i;   theta_i <- h_i
           m_{i -> j_e} <- h_i + sum_{e' != e} r_e'   (e' ascending)   for each e;   publish all deg_i messages

The messages of round k carry exactly ``R_i^k - 1`` models, so
``x_i^(k) = h_i^(k-1) + (1/n) sum_{l != i, d(i,l) <= k} (h_l^(k - d(i,l)) - h_i^(k-1))``, and with full gradients the
fixed point is the minimiser of ``sum_i f_i``.

The early-round weighting is this project's choice: the paper normalises with a relayed count, here the weight of the
models that have not arrived yet goes to the node's own ``h_i``, through the host table ``R_i^k`` (possible because the
tree is fixed).  Round 0 is the identity and from round ``ecc(i)`` on every model has arrived, so the choice has no
effect from then on.

The graph must be a tree (connected, ``n - 1`` undirected edges) and must not change during the run: directed graphs,
link-drop fault injection and a planned graph sequence with more than one topology are refused.  Only the synchronous
(Jacobi) order exists.  The checkpoint carries ``msg``, the messages published at the end of the last round.
"""
from __future__ import annotations

import numpy as np
import torch

from .base import ConsensusOptimizer
from .choco import check_static_plan
from ..ops import consensus_ref as ref


class RelaySum(ConsensusOptimizer):
    alg_name = "relaysum"
    STATE = ("msg",)
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("relaysum runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("relaysum needs a fixed tree: link-drop fault_injection changes the graph during the run")
        graph = self.pr.graph
        if graph.is_directed():
            raise ValueError("relaysum needs an undirected tree (each edge carries a message both ways)")
        self.topo = self.pr.topology()
        if not self.topo.is_tree():
            raise ValueError(f"relaysum needs a tree: the graph has {self.topo.N} nodes, "
                             f"{int(self.topo.adj.sum()) // 2} edges and is "
                             f"{'' if self.topo.is_connected() else 'not '}connected (a tree is connected with "
                             f"n - 1 edges)")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf["mu"])
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        a, pl, t = self.arena, self.pr.placement, self.topo
        self.dmax = max(1, t.max_degree)
        self.reach = t.reach_table()                  # [N, diam + 1] host table R_i^k
        self.diam = self.reach.shape[1] - 1
        rs = t.reverse_slots()
        src_node = np.zeros((pl.L, self.dmax), dtype=np.int64)
        src_slot = np.zeros((pl.L, self.dmax), dtype=np.int64)
        live = np.zeros((pl.L, self.dmax), dtype=bool)
        for l in range(pl.L):
            g = pl.lo + l
            for e, j in enumerate(t.neighbors_noself[g]):
                src_node[l, e], src_slot[l, e], live[l, e] = j, rs[g][e], True
        self._src_node = torch.as_tensor(src_node, device=self.device)
        self._src_slot = torch.as_tensor(src_slot, device=self.device)
        self._live = torch.as_tensor(live, device=self.device)
        # the messages published at the end of the last round: slot e of node i is m_{i -> j_e} (zero past deg_i)
        self.msg = torch.zeros(pl.L, self.dmax, a.n_pad, dtype=a.dtype, device=self.device)

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def reach_m1(self, k: int) -> np.ndarray:
        """``R_i^k - 1`` of the rank's nodes in round k."""
        lo, L = self.pr.placement.lo, self.pr.placement.L
        return self.reach[lo: lo + L, min(k, self.diam)] - 1

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, 1, 0, refresh=self.refresh_graph), "relaysum",
                              "its messages relay over one fixed tree")
            self._plan_checked = True

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        if pr.topology().key != self.topo.key:
            raise ValueError("relaysum needs a fixed tree: the graph changed during the run")
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            msg_all = [pr.gather_rows(self.msg[:, s].contiguous()) for s in range(self.dmax)]
            cm1 = torch.as_tensor(self.reach_m1(k), dtype=a.dtype, device=self.device)
            r = ref.relaysum_mix_(a.theta, msg_all, self._src_node, self._src_slot, self._live, cm1, self.topo.N)
        pr.compute_grads()
        with torch.no_grad():
            ref.relaysum_step_(a.theta, self.msg, r, self._live, a.grad, self.alph)
