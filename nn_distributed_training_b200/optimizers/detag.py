"""DeTAG — gradient tracking with Chebyshev-accelerated multi-step gossip (Lu, De Sa, *Optimal Complexity in
Decentralized Training*, ICML 2021).  No counterpart in the reference.

Every other algorithm here gossips at most once per gradient step.  DeTAG gossips ``gossip_steps`` (K) times per
gradient step, which pays when the graph mixes slowly (``lam`` close to 1).  ``W`` is the Metropolis matrix and
``lam = max |eig(W - 11^T / N)|``.  At the end of round k - 1 node i published ``z_i = theta_i - alpha y_i`` and ``y_i``.
Round k of node i, in this engine's mix-first order:

    X_0 = z, Y_0 = y                                   (every node's rows, as published)
    for s = 0 .. K-1:
        M_s = sum_j W_ij X_s,j                         (own term first, then the neighbors)
        X_{s+1} = X_{s-1} + w_s (M_s - X_{s-1})        (w_s = 1: X_{s+1} = M_s, and X_{s-1} is not read)
        the same recursion for Y
    theta_i = X_K;  g_i = grad loss_i(theta_i)         (one minibatch draw per round)
    y_i = Y_K + (g_i - g_i^old);  g_i^old = g_i;  publish z_i = theta_i - alpha y_i and y_i

The weights are the Chebyshev semi-iterative schedule, computed on the host in float64 from ``lam`` of the fixed graph
(``consensus_ref.chebyshev_weights``): ``w_0 = 1``, ``w_1 = 2 / (2 - lam^2)`` and ``w_s = 1 / (1 - lam^2 w_{s-1} / 4)``.
``accelerate: false`` sets every ``w_s = 1``, which is plain K-step gossip.  K = 1 is DSGT with ``init_grads: false`` in
both modes.

This deviates from the paper on purpose.  DeTAG's accelerated gossip uses one constant momentum
``eta = (1 - sqrt(1 - lam^2)) / (1 + sqrt(1 - lam^2))`` with ``X_{-1} = X_0``.  The schedule above converges to that
constant (``w_inf = 1 + eta``) and is optimal at every K: its worst-case contraction of the disagreement is exactly
``1 / T_K(1 / lam)`` (T_K the Chebyshev polynomial), and it never expands it.  The constant-eta form can expand it: on a
32-node cycle at K = 1 its worst case is 1.30.

W is doubly stochastic and every sub-step is an affine combination with weights summing to 1, so each sub-step keeps
the node mean of X and of Y, and ``sum_i y_i = sum_i g_i`` after every round, to rounding.  ``y`` and ``g_old`` start at
zero, as in K-GT and BEER, so no initial gradient is drawn.

Between rounds theta is the model the last gradient was taken at.  The checkpoint carries ``y``, ``g_old`` and ``z``
(the published row).  Chebyshev acceleration on a changing W has no guarantee, so the graph must be undirected and
fixed: directed graphs, link-drop fault injection and a planned graph sequence with more than one topology are refused;
only the synchronous (Jacobi) order exists.  ``lam`` (``opt.lam``) and the schedule (``opt.omega``) are computed once
from the full matrix, so they are identical on every rank.
"""
from __future__ import annotations

import math
import numbers

import torch

from .base import ConsensusOptimizer
from .choco import check_static_plan
from ..ops import consensus_ref as ref


def check_gossip_steps(v) -> int:
    """``gossip_steps`` must be an integer >= 1 (a bool or a float is refused)."""
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or int(v) < 1:
        raise ValueError(f"detag gossip_steps must be an integer >= 1 (got {v!r})")
    return int(v)


class DeTAG(ConsensusOptimizer):
    alg_name = "detag"
    STATE = ("y", "g_old", "z")

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("detag runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("detag needs a fixed graph: link-drop fault_injection changes the graph during the run "
                             "(Chebyshev acceleration has no guarantee on a changing mixing matrix)")
        if self.pr.graph.is_directed():
            raise ValueError("detag needs an undirected graph (a doubly stochastic Metropolis matrix)")
        if conf.get("byzantine") is not None:
            raise ValueError("detag does not model Byzantine attackers (clipped_gossip and bridge do)")
        self.alpha = float(conf["alpha"])
        if not (math.isfinite(self.alpha) and self.alpha > 0.0):
            raise ValueError(f"detag alpha must be finite and > 0 (got {conf['alpha']!r})")
        self.gossip_steps = check_gossip_steps(conf["gossip_steps"])
        acc = conf.get("accelerate", True)
        if not isinstance(acc, bool):
            raise ValueError(f"detag accelerate must be true or false (got {acc!r})")
        self.accelerate = acc
        self.refresh_graph = bool(conf.get("update_graph", True))
        self.topo = self.pr.topology()
        self.lam = ref.mixing_lambda(self.topo.W)
        self.omega = ref.chebyshev_weights(self.lam, self.gossip_steps, self.accelerate)
        a = self.arena
        self.y = a.zeros()                          # the published tracker of the last round
        self.g_old = a.zeros()
        self.z = a.theta.detach().clone()           # the published theta - alpha y (y = 0 at the start)

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, 1, 0, refresh=self.refresh_graph), "detag",
                              "Chebyshev acceleration has no guarantee on a changing mixing matrix")
            self._plan_checked = True

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        if topo.key != self.topo.key:
            raise ValueError("detag needs a fixed graph: the graph changed during the run")
        w_rows = self._rows(topo, topo.W)
        with torch.no_grad():
            x, y, x_prev, y_prev = self.z, self.y, None, None
            for s, om in enumerate(self.omega):
                xn = ref.ag_gossip(pr.gather_rows(x), x_prev, w_rows, om)
                yn = ref.ag_gossip(pr.gather_rows(y), y_prev, w_rows, om)
                x, y, x_prev, y_prev = xn, yn, x, y
            a.theta.copy_(x)
        pr.compute_grads()
        with torch.no_grad():
            self.z.copy_(ref.detag_track_(self.y, self.g_old, y, a.grad, a.theta, self.alpha))
