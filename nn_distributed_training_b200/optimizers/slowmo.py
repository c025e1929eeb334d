"""SlowMo — slow momentum over the periodic global average of Gossip-PGA and local SGD (Wang, Tantia, Ballas, Rabbat,
*SlowMo: Improving Communication-Efficient Distributed SGD with Slow Momentum*, ICLR 2020).  No counterpart in the
reference.

Gossip-PGA's round (optimizers/gossip_pga.py) with the same index choice: round k is global when
k mod period == period - 1.  Every node also keeps an anchor a_i (theta_i^0 before round 0) and a slow momentum u_i
(0 before round 0).  With DSGD's schedule alpha_k = alpha_{k-1} (1 - mu alpha_{k-1}), round k of node i is

    gossip round:  theta~_i = sum_j W_ij theta_j^k     (gossip: true, DSGD's Metropolis mix)
                   theta~_i = theta_i^k                (gossip: false, local SGD)
    global round:  xbar     = (1/N) sum_j theta_j^k    (pga_mean_: accumulated in fp64, cast once)
                   gamma    = alpha_{k-1}              (alpha_{-1} := alpha0)
                   u_i      <- beta_s u_i + (a_i - xbar) / gamma
                   a_i      <- a_i - alpha_s gamma u_i
                   theta~_i = a_i
                   m_i      <- 0                       (base_momentum > 0 only)
    then:          g_i = grad f_i(theta~_i)
                   base_momentum == 0:  theta_i^{k+1} = theta~_i - alpha_k g_i                  (DSGD's step)
                   base_momentum  > 0:  m_i <- beta_b m_i + g_i
                                        theta_i^{k+1} = theta~_i - alpha_k (nesterov ? g_i + beta_b m_i : m_i)

with beta_s = ``slow_momentum``, alpha_s = ``slow_lr`` and beta_b = ``base_momentum``.  The outer update is evaluated in
fp64 from the stored xbar, a_i and u_i, and each stored row is rounded once (ops/consensus_ref.py: slowmo_outer_).

Where this departs from the paper:
- gamma is alpha_{k-1}, the step of the last base step that fed the average.  The paper holds gamma_t constant within
  an outer iteration; with ``mu = 0`` the two are the same.
- The first outer iteration has period - 1 base steps, not period: Gossip-PGA's index choice.  With ``period == 1``
  round 0 is global with u = 0, so theta~ = theta^0.
- The base momentum buffer is reset to zero at every global round, one of the paper's three buffer policies and the
  only one offered.  A zeroed m makes the next momentum step behave exactly like DSGDm's round-0 step.
- The problems deep-copy one base model into every node, so a_i, u_i and theta~_i are bitwise equal across nodes after
  every global round.  They are still stored per node, as arena rows, so checkpoints and multi-rank placement stay
  generic.

Exact relations: ``period > outer_iterations`` never averages and is DSGD (``base_momentum: 0``) or DSGDm with local
momentum and the same beta and nesterov, bit for bit.  ``slow_momentum: 0, slow_lr: 1`` is Gossip-PGA up to the outer
update's rounding: a - gamma ((a - xbar) / gamma) in fp64 can miss xbar's last bit.

gamma divides, so a schedule that reaches alpha_k <= 0 within ``outer_iterations`` is refused.  The rest is Gossip-PGA's:
changing graphs and link drops affect gossip rounds only; directed graphs, ``mixing_order: reference`` and Byzantine
attackers are refused; on more than one rank the global round needs NVLS.
"""
from __future__ import annotations

import math

import torch

from .gossip_pga import GossipPGA
from ..ops import consensus_ref as ref


def _unit(v, key: str) -> float:
    """A coefficient in [0, 1)."""
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not 0.0 <= float(v) < 1.0:
        raise ValueError(f"slowmo {key} must be in [0, 1) (got {v!r})")
    return float(v)


class SlowMo(GossipPGA):
    alg_name = "slowmo"
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        super().__init__(ddl_problem, device, conf)
        if not self.alph0 > 0.0:
            raise ValueError(f"slowmo alpha0 must be > 0: it is the slow step's gamma of round 0 (got {conf['alpha0']!r})")
        for k, a in enumerate(self.alpha_table()):      # gamma = alpha_{k-1} divides the displacement
            if not a > 0.0:
                raise ValueError(f"slowmo needs every step size > 0, but round {k} has alpha = {a!r} (alpha0 = "
                                 f"{self.alph0}, mu = {self.mu})")
        self.slow_momentum = _unit(conf["slow_momentum"], "slow_momentum")
        self.slow_lr = conf.get("slow_lr", 1.0)
        if isinstance(self.slow_lr, bool) or not isinstance(self.slow_lr, (int, float)) or not (
                math.isfinite(self.slow_lr) and self.slow_lr > 0.0):
            raise ValueError(f"slowmo slow_lr must be finite and > 0 (got {self.slow_lr!r})")
        self.slow_lr = float(self.slow_lr)
        self.base_momentum = _unit(conf.get("base_momentum", 0.0), "base_momentum")
        self.nesterov = conf.get("nesterov", False)
        if not isinstance(self.nesterov, bool):
            raise ValueError(f"slowmo nesterov must be true or false (got {self.nesterov!r})")
        self.anchor = self.arena.theta.detach().clone()
        self.u = self.arena.zeros()
        self.m = self.arena.zeros() if self.base_momentum > 0.0 else None
        self.STATE = ("anchor", "u", "m") if self.m is not None else ("anchor", "u")

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:      # every round, so a link-drop sequence is the one the fused plan draws
            pr.update_graph()
        alpha_prev = self.alph
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            if self.is_global(k):
                ref.pga_mean_(a.theta, pr.gather_rows(a.theta))
                ref.slowmo_outer_(a.theta, self.anchor, self.u, self.m, alpha_prev, self.slow_lr, self.slow_momentum)
            elif self.gossip:
                topo = pr.topology()
                a.theta.copy_(ref.dsgd_mix(pr.gather_rows(a.theta), self._rows(topo, topo.W)))
        pr.compute_grads()
        with torch.no_grad():
            if self.m is None:
                ref.dsgd_step_(a.theta, a.grad, self.alph)
            else:
                ref.dsgdm_step_(a.theta, self.m, None, a.grad, self.alph, alpha_prev, self.base_momentum, False,
                                self.nesterov, k == 0)
