"""Push-DIGing — gradient tracking on push-sum gossip (Nedić, Olshevsky, Shi, SIAM J. Optim. 2017; with stochastic
gradients the setting of S-ADDOPT, Qureshi, Xin, Khan 2021).  No counterpart in the reference.

DSGT corrects DSGD's bias on heterogeneous data but needs a doubly stochastic matrix; SGP runs on directed graphs but
carries DSGD's bias.  Push-DIGing does both: it mixes with SGP's column-stochastic push weights
``A_ij = 1 / (d_out(j) + 1)`` for ``j -> i`` and ``j = i`` (``Topology.push_weights``) and tracks the network's average
gradient as DSGT does.  It is proven for time-varying directed graphs.  With a constant step ``alpha``, round k of
node i is

    mix:    u_i <- sum_{j in in_k(i) + i} A_ij (u_j - alpha y_j)^pub
            w_i <- sum A_ij w_j^pub  (float64)        theta_i <- u_i / w_i
    track:  y_i <- sum A_ij y_j^pub + g_i - g_old_i   (g_i = grad loss_i(theta_i))
            g_old_i <- g_i;  publish (u_i, w_i) and y_i

starting from ``u = theta0``, ``w = 1``, ``y = 0``, ``g_old = 0``: round 0 only mixes, and since A preserves column
sums, ``sum_i y_i = sum_i g_i`` from the first track on.  (There is no ``init_grads``: the zero start needs no extra
gradient draw.)  Between rounds ``theta = u / w`` is the model that evaluation, checkpoints and the metrics see.  On the
undirected cycle the push weights are the Metropolis weights, ``w`` stays 1 and Push-DIGing is DSGT with
``init_grads: false``.  Only the synchronous (Jacobi) order exists.
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class PushDIGing(ConsensusOptimizer):
    alg_name = "push_diging"
    STATE = ("u", "w", "y", "g")

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("push_diging runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        g = getattr(self.pr, "graph", None)
        if pconf.get("fault_injection") and g is not None and g.is_directed():
            raise ValueError("push_diging: link-drop fault_injection drops undirected edges and does not apply to a "
                             "directed graph")
        self.alpha = float(conf["alpha"])
        self.refresh_graph = bool(conf.get("update_graph", True))
        a = self.arena
        self.u = a.theta.detach().clone()
        self.w = torch.ones(a.L, dtype=torch.float64, device=self.device)
        self.y = a.zeros()
        self.g = a.zeros()             # g_old
        self.ysum = a.zeros()          # sum_j A_ij y_j of the current round (scratch between mix and track)

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        with torch.no_grad():
            u_all = pr.gather_rows(self.u)
            y_all = pr.gather_rows(self.y)
            w_all = pr.gather_rows(self.w.view(-1, 1)).view(-1)
            ref.pdg_mix_(self.u, self.w, a.theta, self.ysum, u_all, y_all, w_all,
                         self._rows(topo, topo.push_weights), self.alpha)
        pr.compute_grads()
        with torch.no_grad():
            ref.pdg_track_(self.y, self.g, self.ysum, a.grad)
