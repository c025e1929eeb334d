"""Exact Diffusion — bias-corrected diffusion (Yuan, Ying, Zhao, Sayed, IEEE TSP 2019; the same recursion as D²,
Tang et al. 2018).  No counterpart in the reference.

With ``A = (I + W) / 2`` the Metropolis matrix averaged with the identity and DSGD's step schedule
``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})``, round k of node i is

    mix:      theta_i <- sum_j A_ij theta_j^pub         (combine; theta_j^pub published at the end of round k-1)
    round 0:  psi_i   <- theta_i
    adapt:    psi'    =  theta_i - alpha_k grad loss_i(theta_i)
    correct:  theta_i <- psi' + (theta_i - psi_i);  psi_i <- psi';  publish theta_i

Like DSGD it publishes one row per round; it keeps one more local row (psi), and unlike DSGD it converges to the
exact minimiser of the summed losses on a static graph with a constant step when node data differ.  Between rounds
theta holds the value before the mix, as it does for DSGD.  Only the synchronous (Jacobi) order exists.
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class ExactDiffusion(ConsensusOptimizer):
    alg_name = "exact_diffusion"
    STATE = ("psi",)
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("exact_diffusion runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        self.psi = self.arena.zeros()

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
            theta_all = pr.gather_rows(a.theta)
            a.theta.copy_(ref.dsgd_mix(theta_all, self._rows(topo, ref.ed_weights(topo.W))))
            if k == 0:
                self.psi.copy_(a.theta)
        pr.compute_grads()
        with torch.no_grad():
            ref.ed_step_(a.theta, self.psi, a.grad, self.alph)
