"""ClippedGossip — Byzantine-robust gossip (He, Karimireddy, Jaggi, *Byzantine-robust decentralized learning via
ClippedGossip*, 2022), and DSGD under attack with ``clip: none``.  No counterpart in the reference.

DSGD's step schedule (``alpha0``, ``mu``) and single published channel.  Round k of node i, in this engine's mix-first
order (``theta_j^pub`` is the row node j published at the end of round k-1):

    dist:   d_ij = |theta_j^pub - theta_i|_2 for every neighbor j               (fp64)
    radius: the neighbors by decreasing d_ij (ties: smaller index first); the leading ones whose Metropolis weights
            sum to at most delta are clipped, tau_i = d of the first one that does not fit (0 if all fit)
    mix:    theta_i <- theta_i + sum_j W_ij min(1, tau_i / d_ij) (theta_j^pub - theta_i)
    step:   theta_i <- theta_i - alpha_k grad loss_i(theta_i); publish theta_i

With ``clip: none`` the mix is DSGD's ``sum_j W_ij theta_j^pub`` (own term theta_i).  Byzantine nodes
(``byzantine: {nodes, attack, scale, z}``) run the same update on their own row and publish, in place of theta_i,
``-scale theta_i`` (``sign_flip``) or ``mu - z sigma`` of their honest neighbors' rows read this round (``alie``,
Baruch, Baruch, Goldberg, NeurIPS 2019).  Every neighbor sees the same published row.

The rows each node last published are optimizer state: an ALIE row cannot be rebuilt from theta, so the checkpoint
carries them and a fused resume publishes them.  Only the synchronous (Jacobi) order on undirected graphs exists;
changing graphs and link drops are allowed (the distances and radii come from each round's graph).
"""
from __future__ import annotations

import math
import numbers
from typing import List

import numpy as np
import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref

CLIP_MODES = ("none", "adaptive")


def check_byzantine(byz, N: int) -> List[int]:
    """The validated, sorted Byzantine node ids of ``byzantine`` for a graph of N nodes (``ValueError`` naming the
    reason otherwise)."""
    if not isinstance(byz, dict):
        raise ValueError(f"byzantine must be a mapping with nodes and attack (got {byz!r})")
    if byz.get("attack") not in ref.ATTACK_CODE:
        raise ValueError(f"byzantine.attack must be one of {'|'.join(ref.ATTACK_CODE)} (got {byz.get('attack')!r})")
    nodes = byz.get("nodes")
    if not isinstance(nodes, (list, tuple)) or not nodes or any(
            isinstance(v, bool) or not isinstance(v, numbers.Integral) for v in nodes):
        raise ValueError(f"byzantine.nodes must be a non-empty list of node ids (got {nodes!r})")
    nodes = [int(v) for v in nodes]
    if len(set(nodes)) != len(nodes):
        raise ValueError(f"byzantine.nodes has duplicated node ids ({nodes})")
    if N is not None:
        bad = [v for v in nodes if not 0 <= v < N]
        if bad:
            raise ValueError(f"byzantine.nodes {bad} out of range for a graph of {N} nodes")
        if len(nodes) >= N:
            raise ValueError(f"byzantine.nodes cover every node of the graph ({N}): no honest node is left")
    for key in ("scale", "z"):
        v = byz.get(key, 1.0)
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)):
            raise ValueError(f"byzantine.{key} must be a finite number (got {v!r})")
    return sorted(nodes)


def setup_attackers(opt, byz) -> None:
    """The attacker fields of a Byzantine-robust optimizer (ClippedGossip, BRIDGE) from ``byzantine`` (or None):
    ``byzantine`` (sorted node ids), ``attack_name``, ``scale``, ``z`` and ``attack``, the attack code of each local
    node (cg_step's table)."""
    attacked = byz is not None
    opt.byzantine = check_byzantine(byz, opt.pr.N) if attacked else []
    opt.attack_name = byz["attack"] if attacked else None
    opt.scale = float(byz.get("scale", 1.0)) if attacked else 1.0
    opt.z = float(byz.get("z", 1.0)) if attacked else 1.0
    lo, L = opt.pr.placement.lo, opt.pr.placement.L
    code = ref.ATTACK_CODE.get(opt.attack_name, 0)
    opt.attack = [code if lo + l in opt.byzantine else 0 for l in range(L)]    # per local node


class ClippedGossip(ConsensusOptimizer):
    alg_name = "clipped_gossip"
    STATE = ("pub",)
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("clipped_gossip runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and hasattr(graph, "is_directed") and graph.is_directed():
            raise ValueError("clipped_gossip needs an undirected graph (a doubly stochastic Metropolis matrix)")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.alph = self.alph0
        self.clip = conf["clip"]
        if self.clip not in CLIP_MODES:
            raise ValueError(f"clipped_gossip clip must be one of {'|'.join(CLIP_MODES)} (got {self.clip!r})")
        self.delta = float(conf["delta"]) if self.clip == "adaptive" else 0.0
        if self.clip == "adaptive" and not 0.0 <= self.delta < 1.0:
            raise ValueError(f"clipped_gossip delta must be in [0, 1) (got {conf['delta']!r})")
        self.refresh_graph = bool(conf.get("update_graph", True))
        setup_attackers(self, conf.get("byzantine"))
        self.pub = self.arena.theta.detach().clone()      # the rows the local nodes published last

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``), DSGD's schedule."""
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
        lo = pr.placement.lo
        with torch.no_grad():
            pub_all = pr.gather_rows(self.pub)
            if self.clip == "adaptive":
                # the weights rounded to the row dtype, as the kernels' tables hold them
                W = topo.W.astype(np.float32 if a.dtype == torch.float32 else np.float64)
                ref.cg_mix_(a.theta, pub_all, W, topo.neighbors_noself, lo, self.delta)
            else:
                w_rows = self._rows(topo, topo.W)
                mixed = ref.dsgd_mix(pub_all, w_rows)
                for l, code in enumerate(self.attack):
                    if code:      # the own term of a Byzantine node is its own theta, not the row it published
                        own = pub_all.clone()
                        own[lo + l] = a.theta[l]
                        mixed[l] = w_rows[l] @ own
                a.theta.copy_(mixed)
        pr.compute_grads()
        with torch.no_grad():
            ref.dsgd_step_(a.theta, a.grad, self.alph)
            ref.cg_publish_(self.pub, a.theta, pub_all, self.attack, topo.neighbors_noself, set(self.byzantine), lo,
                            self.scale, self.z)
