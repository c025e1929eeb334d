"""Cross-gradient gossip — every node steps along a weighted mean of gradients from its whole neighbourhood's data
(Cross-Gradient Aggregation, Esfandiari, Tan, Jiang, Balu, Herron, Hegde, Sarkar, ICML 2021; Neighborhood Gradient
Clustering / Mean, Aketi, Kodge, Roy).  No counterpart in the reference.

Heterogeneous data biases DSGD's fixed point towards each node's own minimiser.  Tracking (DSGT) and bias correction
(Exact Diffusion) remove that bias on the model side; cross-gradient methods remove it on the data side: node i also
evaluates its neighbours' models on its own minibatch and sends those gradients back, so each node steps along
gradients from its whole neighbourhood's data.  With ``lam = cross_weight`` in [0, 1] and DSGD's step schedule
``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})``, round k of node i with neighbours ``j_1 .. j_deg`` (table order) is

    xmix_i   = sum_j W_ij x_j^k                           (dsgd_mix's accumulation and rounding)
    g_ii     = grad f_i(x_i^k; xi_i^k)                    (own point, own draw)
    g_{i->j} = grad f_i(x_j^k; xi_i^k)                    for every neighbour j (the SAME draw), sent to j
    d_i      = c0_i g_ii + sum_e (lam W_{i j_e}) g_{j_e->i},   c0_i = (1 - lam) + lam W_ii
               (coefficients and sum in float64, own term first, then table order, rounded once to the arena dtype)
    x_i^{k+1} = xmix_i - alpha_k d_i                       (dsgd_step's arithmetic on (xmix, d)); publish

This is the D-PSGD form (Lian et al., NeurIPS 2017): every gradient is taken at the *published* point x^k, which is what
theta holds between rounds.  With one model publication per round the published row is the only point of node j that
node i can know, so the cross-gradients are taken there.  This repository's DSGD takes its gradient at the mixed point
instead; a cross-gradient at j's mixed point would need a third publication per round.  So ``lam = 0`` is D-PSGD (not
this repository's DSGD), bit for bit, since ``1 g + sum 0 g' = g``.

Deviations from the papers, both deliberate: CGA projects the neighbourhood's gradients with a per-node quadratic
program, and NGC uses momentum; here the aggregate is the plain Metropolis-weighted mean above, with ``lam`` blending
it with the own gradient.  ``lam = 1`` on the complete graph with equal rows is centralized minibatch SGD on the union
of the N minibatches.

The state is theta alone (and DSGD's ``alph``): the cross-gradients of a round are consumed in that round.  The graph
must be undirected and fixed (each edge carries a gradient back to the node whose model it was taken at, through the
reverse slot): directed graphs, link drops and a planned graph sequence of more than one topology are refused, as are
``mixing_order: reference``, Byzantine attackers and a problem driven through the reference's API
(``ReferenceProblemAdapter``, e.g. PPO), which draws its minibatch internally and cannot evaluate it at several points.
A round costs ``1 + dmax`` forward/backward passes per node (``dmax`` the largest degree; a node of lower degree computes
its idle slots at its own row and publishes nothing for them), of which ``N + 2|E|`` over the network are used.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .base import ConsensusOptimizer, ReferenceProblemAdapter
from .choco import check_static_plan
from ..ops import consensus_ref as ref


def check_cross_weight(v) -> float:
    """``cross_weight`` must be finite and in [0, 1] (a bool is refused)."""
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not (math.isfinite(float(v)) and 0.0 <= float(v) <= 1.0):
        raise ValueError(f"cross_gradient cross_weight must be finite and in [0, 1] (got {v!r})")
    return float(v)


class CrossGradient(ConsensusOptimizer):
    alg_name = "cross_gradient"
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("cross_gradient runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        if isinstance(self.pr, ReferenceProblemAdapter):
            raise ValueError("cross_gradient needs gradients at several points on the same minibatch, and a problem "
                             "driven through the reference API (local_batch_loss, e.g. the PPO problem) draws its batch "
                             "internally and cannot evaluate it at another point")
        if conf.get("byzantine") is not None:
            raise ValueError("cross_gradient does not model Byzantine attackers (clipped_gossip and bridge do)")
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("cross_gradient needs a fixed graph: link-drop fault_injection changes it during the run")
        if self.pr.graph.is_directed():
            raise ValueError("cross_gradient needs an undirected graph (each edge carries a gradient back to the node "
                             "whose model it was taken at)")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        for name, v in (("alpha0", self.alph0), ("mu", self.mu)):
            if not (math.isfinite(v) and v >= 0.0):
                raise ValueError(f"cross_gradient {name} must be finite and >= 0 (got {v!r})")
        self.lam = check_cross_weight(conf["cross_weight"])
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        from ..ops.engine import check_wait_capacity
        a, pl, t = self.arena, self.pr.placement, self.pr.topology()
        self.topo = t
        self.dmax = max(1, t.max_degree)
        check_wait_capacity(self.dmax, 0)
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
        coef0, coef = ref.xg_coefs(t.W, t.neighbors_noself, self.lam, pl.lo, pl.L, self.dmax)
        self.coef0 = torch.as_tensor(coef0, device=self.device)
        self.coef = torch.as_tensor(coef, device=self.device)
        # the cross points of the round and (PyTorch path) the gradients there: [dmax, L, n_pad]
        self.theta_x = torch.zeros(self.dmax, pl.L, a.n_pad, dtype=a.dtype, device=self.device)
        self.grad_x = torch.zeros_like(self.theta_x)
        if self.pr.fused is not None:               # one more forward/backward op per neighbour slot
            self.pr.fused.enable_cross_points(self.theta_x)
        useful, launched = self.grad_evals()
        # saved with the metrics (<problem>_results.pt): what a round costs against DSGD's N evaluations
        self.pr.xg_grad_evals = {"useful_per_round": useful, "launched_per_round": launched, "rounds": self.oits}

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def grad_evals(self):
        """Gradient evaluations per round over the network: ``(useful, launched)`` = ``(N + 2|E|, N (1 + dmax))``."""
        t = self.topo
        return t.N + int(t.adj.sum()), t.N * (1 + self.dmax)

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, 1, 0, refresh=self.refresh_graph),
                              "cross_gradient", "its cross-gradients travel back over the edges of one fixed graph")
            self._plan_checked = True

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        if pr.topology().key != self.topo.key:
            raise ValueError("cross_gradient needs a fixed graph: the graph changed during the run")
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            theta_all = pr.gather_rows(a.theta)
            xmix = ref.dsgd_mix(theta_all, self._rows(self.topo, self.topo.W))
            self.theta_x.copy_(ref.xg_cross_points(theta_all, self._src_node, self._live, pr.placement.lo))
        pr.compute_grads_multi(self.theta_x, self.grad_x)
        with torch.no_grad():
            gx_all = torch.stack([pr.gather_rows(self.grad_x[e]) for e in range(self.dmax)])
            recv = ref.xg_received(gx_all, self._src_node, self._src_slot, self._live)
            ref.xg_step_(a.theta, xmix, a.grad, recv, self.coef0, self.coef, self.alph)
