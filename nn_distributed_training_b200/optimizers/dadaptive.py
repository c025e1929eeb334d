"""Decentralized adaptive gradient methods with a gossiped second moment: decentralized AMSGrad and decentralized
AdaGrad (Chen, Karimi, Zhao, Li, *On the Convergence of Decentralized Adaptive Gradient Methods*, ACML 2022).  No
counterpart in the reference.

If every node runs DSGD and divides by its own second moment (DADAM-style), the run converges to a point where
``sum_i g_i / sqrt(v_i) = 0`` instead of ``sum_i g_i = 0``; whenever the nodes see different gradient scales that point
is not stationary, and a smaller step does not move it.  The fix gossips a tracker ``u~_i`` of the second moment beside
the parameters, so every node divides by (nearly) the same network-wide estimate.  With a constant step ``alpha``,
round k of node i on the graph W_k (Metropolis, doubly stochastic) is, in this engine's mix -> gradient -> step order,

    mix:   x_i <- sum_j W_ij theta_j^pub            z_i <- sum_j W_ij u~_j^pub     (tracking only)
    fwd/bwd at x_i: g_i
    step:  m_i <- beta1 m_i + (1 - beta1) g_i
           amsgrad:  v_i <- beta2 v_i + (1 - beta2) g_i^2;   vhat'_i = max(vhat_i, v_i)
           adagrad:  vhat'_i = vhat_i + (g_i^2 - vhat_i) / (k + 1)       (running mean of g^2 over rounds 0..k)
           tracking: u~_i <- z_i + (vhat'_i - vhat_i);   u_i = max(u~_i, eps)
           own:      u_i = max(vhat'_i, eps)
           vhat_i <- vhat'_i;   theta_i <- x_i - alpha m_i / sqrt(u_i);   publish theta_i (and u~_i)

The state starts at m = 0, v = 0 and vhat = eps on every element (padding included); with tracking the published
tracker of round 0 is u~ = eps, so ``sum_i u~_i = sum_i vhat_i`` from the start and, W_k being doubly stochastic, after
every round for any sequence of graphs: changing graphs and link drops are allowed, as for K-GT.

Two deliberate departures from the paper's Algorithm 1:
- The denominator includes the node's own increment of this round, as Adam's does.  Taken literally, the paper
  divides round 1 by u = eps, a first step of alpha (1 - beta1) g / sqrt(eps): 1000 alpha g at eps = 1e-8, which
  blows up a neural network.
- There is no bias correction, as in the paper.

Between rounds theta is the published row (as for DSGD).  The checkpoint carries m and vhat, plus v (amsgrad) and the
tracker u~ (tracking); AdaGrad's count is the round index k.  Only the synchronous (Jacobi) order on undirected graphs
exists: the tracker needs a doubly stochastic W.
"""
from __future__ import annotations

import math

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class DAdaptive(ConsensusOptimizer):
    alg_name = "dadaptive"

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("dadaptive runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and hasattr(graph, "is_directed") and graph.is_directed():
            raise ValueError("dadaptive needs an undirected graph (a doubly stochastic Metropolis matrix)")
        self.alpha = float(conf["alpha"])
        if not self.alpha > 0.0:
            raise ValueError(f"dadaptive alpha must be > 0 (got {conf['alpha']!r})")
        self.variant = conf["variant"]
        if self.variant not in ref.DADAPTIVE_VARIANTS:
            raise ValueError(f"dadaptive variant must be one of {'|'.join(ref.DADAPTIVE_VARIANTS)} "
                             f"(got {self.variant!r})")
        self.adagrad = self.variant == "adagrad"
        if self.adagrad and "beta2" in conf:
            raise ValueError("dadaptive beta2 applies to variant amsgrad only")
        self.tracking = bool(conf.get("tracking", True))
        self.beta1 = float(conf.get("beta1", 0.9))
        self.beta2 = float(conf.get("beta2", 0.999))
        self.eps = float(conf.get("eps", 1e-8))
        for name, b in (("beta1", self.beta1), ("beta2", self.beta2)):
            if not 0.0 <= b < 1.0:
                raise ValueError(f"dadaptive {name} must be in [0, 1) (got {b!r})")
        if not (math.isfinite(self.eps) and self.eps > 0.0):
            raise ValueError(f"dadaptive eps must be finite and > 0 (got {conf.get('eps')!r})")
        self.refresh_graph = bool(conf.get("update_graph", True))
        a = self.arena
        self.m = a.zeros()
        self.v = None if self.adagrad else a.zeros()
        self.vhat = a.zeros().fill_(self.eps)
        # the published tracker u~ (between rounds; the fused mix leaves z here until sync_back)
        self.ut = a.zeros().fill_(self.eps) if self.tracking else None
        self.STATE = ("m", "vhat") + (() if self.adagrad else ("v",)) + (("ut",) if self.tracking else ())

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        with torch.no_grad():
            theta_all = pr.gather_rows(a.theta)
            ut_all = pr.gather_rows(self.ut) if self.tracking else None
            ref.dadaptive_mix_(a.theta, self.ut, theta_all, ut_all, self._rows(topo, topo.W))
        pr.compute_grads()
        with torch.no_grad():
            ref.dadaptive_step_(a.theta, self.m, self.v, self.vhat, self.ut, a.grad, self.alpha, self.beta1,
                                self.beta2, self.eps, k, self.adagrad)
