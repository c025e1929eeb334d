"""DSGD — decentralized SGD with Metropolis mixing
(reference: optimizers/dsgd.py:7-62).

    alpha_k   = alpha_{k-1} (1 - mu alpha_{k-1})
    theta~_i  = sum_{j in N_i + i} W_ij theta_j^k
    theta_i^{k+1} = theta~_i - alpha_k grad loss_i(theta~_i)

Default is the synchronous (Jacobi) update — what N concurrently running GPUs
implement.  ``mixing_order: reference`` reproduces the reference's in-place
node-index sweep (Gauss-Seidel, SURVEY Q1) for oracle tests.  The Metropolis
matrix is cached per edge set instead of being rebuilt every round (Q2).
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class DSGD(ConsensusOptimizer):
    alg_name = "dsgd"
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        super().__init__(ddl_problem, device, conf)
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf["mu"])
        self.alph = self.alph0
        # Q6: the reference never refreshes a dynamic graph for DSGD
        self.refresh_graph = bool(conf.get("update_graph", True))

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``)."""
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
            if self.mixing_order == "reference":
                W = torch.as_tensor(topo.W, dtype=a.dtype, device=self.device)
                ref.dsgd_mix_sequential_(a.theta, W, topo.neighbors)
            else:
                theta_all = pr.gather_rows(a.theta)
                a.theta.copy_(ref.dsgd_mix(theta_all, self._rows(topo, topo.W)))
        pr.compute_grads()
        with torch.no_grad():
            ref.dsgd_step_(a.theta, a.grad, self.alph)
