"""DSGD with momentum: local heavy-ball momentum, or quasi-global momentum (QG-DSGDm: Lin, Karimireddy, Stich, Jaggi,
*Quasi-Global Momentum: Accelerating Decentralized Deep Learning on Heterogeneous Data*, ICML 2021), optionally in
Nesterov form.  No counterpart in the reference.

With DSGD's step schedule ``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})``, round k of node i is

    mix:   x_i <- sum_j W_ij theta_j^pub                    (DSGD's mix; theta_j^pub published at the end of round k-1)
    fwd/bwd at x_i: g_i
    local:         m_i <- beta m_i + g_i                                  (m_i = 0 before round 0)
    quasi_global:  if k > 0:  d_i = (x_prev_i - x_i) / alpha_{k-1}
                              mhat_i <- beta mhat_i + (1 - beta) d_i      (mhat_i = 0 before round 0)
                   m_i = beta mhat_i + g_i   (not stored);  x_prev_i <- x_i
    both:          theta_i <- x_i - alpha_k (nesterov ? g_i + beta m_i : m_i);  publish theta_i

Quasi-global momentum replaces the local gradient history by the rows' own displacement between rounds, which after
the mix carries the neighbors' progress too; on heterogeneous data it avoids the drift of local momentum towards each
node's own minimiser.  This is the paper's Algorithm 1 in this engine's mix -> gradient -> step order: its x^(t) is the
mixed row, so d of the paper's iteration t - 1 is formed at the start of the step of round t, before mhat is used.
The paper allows a separate coefficient for mhat's average; here ``beta`` serves both.  Like DSGD it publishes one
row per round; it keeps one local row (m) or two (mhat, x_prev).  Round 0 is a DSGD step, and with ``beta = 0`` every
round is.  Between rounds theta holds the published row, as it does for DSGD.  Only the synchronous (Jacobi) order
exists.
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref

MOMENTUM_MODES = ("local", "quasi_global")


class DSGDm(ConsensusOptimizer):
    alg_name = "dsgdm"
    STATE = ("m",)
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("dsgdm runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.alph = self.alph0
        self.beta = float(conf["beta"])
        if not 0.0 <= self.beta < 1.0:
            raise ValueError(f"dsgdm: beta must be in [0, 1) (got {self.beta!r})")
        if conf["momentum"] not in MOMENTUM_MODES:
            raise ValueError(f"dsgdm: momentum must be one of {'|'.join(MOMENTUM_MODES)} (got {conf['momentum']!r})")
        self.quasi_global = conf["momentum"] == "quasi_global"
        self.nesterov = bool(conf.get("nesterov", False))
        self.refresh_graph = bool(conf.get("update_graph", True))
        if self.quasi_global:
            # alpha_{k-1} divides the displacement of round k
            for k, a in enumerate(self.alpha_table()):
                if not a > 0.0:
                    raise ValueError(f"dsgdm with quasi-global momentum needs every step size > 0, but round {k} has "
                                     f"alpha = {a!r} (alpha0 = {self.alph0}, mu = {self.mu})")
        self.m = self.arena.zeros()
        self.x_prev = self.arena.zeros() if self.quasi_global else None
        if self.quasi_global:
            self.STATE = ("m", "x_prev")

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
        alpha_prev = self.alph
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            theta_all = pr.gather_rows(a.theta)
            a.theta.copy_(ref.dsgd_mix(theta_all, self._rows(topo, topo.W)))
        pr.compute_grads()
        with torch.no_grad():
            ref.dsgdm_step_(a.theta, self.m, self.x_prev, a.grad, self.alph, alpha_prev, self.beta, self.quasi_global,
                            self.nesterov, k == 0)
