"""PowerGossip — rank-one compressed gossip of each edge's model difference (Vogels, Karimireddy, Jaggi, *Practical
Low-Rank Communication Compression in Decentralized Deep Learning*, NeurIPS 2020).  No counterpart in the reference.

Every parameter tensor with two or more dimensions is a matrix ``(shape[0], prod(shape[1:]))`` (``PgLayout``); the
1-D tensors (biases) are gossiped whole.  For each edge ``e = {lo, hi}`` (``lo < hi``) and matrix l both endpoints hold
a unit row-space vector ``p_{e,l}`` (length m_l) and a unit column-space vector ``q_{e,l}`` (length n_l), drawn at
construction from ``np.random.default_rng((lo, hi, l))`` and carried from round to round (warm-started power
iteration).  Nothing of this state depends on which endpoint holds it, and there is no error-feedback row.

Round k runs phase ``k & 1``: phase 0 uses q, phase 1 uses p.  ``W`` are the Metropolis weights, ``gamma`` is in
(0, 1], ``s_{i,e}`` is +1 when ``i = lo`` else -1, and ``alpha_k`` is DSGD's schedule.  Between rounds ``theta_i``
holds h_i and node i has published one message per neighbor.  Round k of node i, in this engine's mix -> gradient ->
step order:

    mix:   per edge e (ascending slot order), per matrix l, with M = X_lo - X_hi:
             d = a_lo - a_hi          (the two endpoints' published products: the same bits at both ends)
             phase 0:  d = M q;    U_e = d q^T;    p_{e,l} <- d / |d|
             phase 1:  d = M^T p;  U_e = p d^T;    q_{e,l} <- d / |d|
           (|d| in float64 in one fixed order, one rounding; |d| = 0 keeps the stored vector)
           x_i = h_i - gamma sum_e W_ie s_ie U_e       (matrix elements)
           x_i = h_i - gamma sum_e W_ie (h_i - h_j)    (1-D tensors, from the messages' bias blocks)
    fwd/bwd at x_i: g_i
    step:  h_i = x_i - alpha_k g_i;   publish msg_{i->e} = [per matrix h_i v | h_i's 1-D tensors]
           (v = the vector of phase (k + 1) & 1)

``U_e`` is the orthogonal projection of ``M`` onto a rank-one subspace and node lo subtracts the ``W U_e`` node hi
adds, so ``sum_i x_i = sum_i h_i`` to rounding; at ``alpha = 0`` the consensus distance never increases.  In phase 1 a
layer whose difference is exactly rank one is removed exactly (two nodes at ``gamma = 1`` land on the midpoint), and
when every parameter is 1-D and ``gamma = 1`` the method is DSGD.

The paper runs both power-iteration half-steps in every round, with two exchanges.  Alternating them, one half-step
per round, is this project's choice: a round keeps one publication, and every neighbor read stays in the round's first
kernel.  Only rank one is implemented.

The graph must be undirected and fixed: directed graphs, link-drop fault injection and a planned graph sequence with
more than one topology are refused; only the synchronous (Jacobi) order exists.  The checkpoint carries ``vec`` (every
edge's vectors) and ``msg`` (the messages published at the end of the last round).
"""
from __future__ import annotations

import numpy as np
import torch

from .base import ConsensusOptimizer
from .choco import check_static_plan
from ..ops import consensus_ref as ref


class PowerGossip(ConsensusOptimizer):
    alg_name = "powergossip"
    STATE = ("vec", "msg")
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("powergossip runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("powergossip needs a fixed graph: link-drop fault_injection changes the graph during the "
                             "run (both endpoints of an edge carry its vectors from round to round)")
        if self.pr.graph.is_directed():
            raise ValueError("powergossip needs an undirected graph (both endpoints of an edge compress the same "
                             "difference)")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.gamma = float(conf["gamma"])
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        a, pl = self.arena, self.pr.placement
        t = self.topo = self.pr.topology()
        self.lay = ref.PgLayout(a.layout)
        self.dmax = max(1, t.max_degree)
        rs = t.reverse_slots()
        src_node = np.zeros((pl.L, self.dmax), dtype=np.int64)
        src_slot = np.zeros((pl.L, self.dmax), dtype=np.int64)
        live = np.zeros((pl.L, self.dmax), dtype=bool)
        sign = np.zeros((pl.L, self.dmax), dtype=np.int32)
        w = np.zeros((pl.L, self.dmax))
        # every edge's vectors: slot e of node i holds those of edge {i, j_e}
        self.vec = torch.zeros(pl.L, self.dmax, self.lay.P + self.lay.Q, dtype=a.dtype, device=self.device)
        for l in range(pl.L):
            g = pl.lo + l
            for e, j in enumerate(t.neighbors_noself[g]):
                src_node[l, e], src_slot[l, e], live[l, e] = j, rs[g][e], True
                sign[l, e] = 1 if g < j else -1
                w[l, e] = t.W[g, j]
                self.vec[l, e] = ref.pg_start_vectors(self.lay, min(g, j), max(g, j), a.dtype)
        self._src_node = torch.as_tensor(src_node, device=self.device)
        self._src_slot = torch.as_tensor(src_slot, device=self.device)
        self._live = torch.as_tensor(live, device=self.device)
        self.sign = torch.as_tensor(sign, device=self.device)
        self._w = torch.as_tensor(w, dtype=a.dtype, device=self.device)
        # the messages published for round 0: products with the phase-0 vectors q
        self.msg = ref.pg_messages(a.theta, self.vec, self._live, self.lay, 0)

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, 1, 0, refresh=self.refresh_graph), "powergossip",
                              "both endpoints of an edge carry its power-iteration vectors from round to round")
            self._plan_checked = True

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        if pr.topology().key != self.topo.key:
            raise ValueError("powergossip needs a fixed graph: the graph changed during the run")
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            msg_all = torch.stack([pr.gather_rows(self.msg[:, s].contiguous()) for s in range(self.dmax)])
            nbr = msg_all[self._src_slot, self._src_node]
            ref.pg_mix_(a.theta, self.vec, self.msg, nbr, self.sign, self._w, self._live, self.gamma, self.lay, k & 1)
        pr.compute_grads()
        with torch.no_grad():
            ref.pg_step_(a.theta, self.msg, a.grad, self.alph, self.vec, self._live, self.lay, (k + 1) & 1)
