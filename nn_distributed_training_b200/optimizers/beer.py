"""BEER — gradient tracking with compressed gossip (Zhao, Li, Li, Richtárik, Chi, NeurIPS 2022).  No counterpart in the
reference.

CHOCO-SGD compresses gossip but keeps DSGD's bias on heterogeneous data; DSGT removes the bias but pulls two full rows
per edge.  BEER is DSGT's gradient tracking with both the parameters and the tracker gossiped through CHOCO's
compressed differences (error feedback through public estimates).  Each node publishes two code rows per round, in
CHOCO's formats and byte layouts (``compressor``: ``none``, ``int8``, ``sign`` or ``topk`` with ``topk_ratio``,
``ops/consensus_ref.py``).  Node i
keeps ``theta`` (x), ``h`` (public estimate of x: the sum of its decoded x-codes), ``s_h = sum_j W_ij h_j``, the tracker
``v``, ``g`` (public estimate of v), ``s_g = sum_j W_ij g_j`` (own terms included) and ``m_old``, the previous round's
gradient.  With a constant step ``alpha`` (the paper's eta) and the consensus step ``gamma`` in (0, 1], round k is

    mix:   s_h_i += W_ii dec(qh_i) + sum_j W_ij dec(qh_j)    s_g_i += W_ii dec(qg_i) + sum_j W_ij dec(qg_j)
           theta_i += gamma (s_h_i - h_i) - alpha v_i        (the codes published at the end of round k-1; zero in round 0)
    step:  v_i += gamma (s_g_i - g_i) + grad_i - m_old_i;  m_old_i <- grad_i      (grad_i = grad loss_i(theta_i))
           qh_i = Q(theta_i - h_i); h_i += dec(qh_i);  qg_i = Q(v_i - g_i); g_i += dec(qg_i);  publish (qh_i, qg_i)

State convention (checkpoints and the fused engine rely on it): between rounds ``h`` and ``g`` include the pending codes,
``s_h`` and ``s_g`` do not, and the pending code rows are ``code_h`` and ``code_g``.  Everything starts at zero, so
round 0 does not move theta and ``sum_i v_i = sum_i m_old_i`` holds from the first step on.  The paper starts the
tracker from a first gradient instead; this zero start needs no extra gradient draw (as Push-DIGing).  With
``compressor: none``, ``gamma: 1`` and a common starting row the iterates are DSGT's with ``own_tracker_step: true,
init_grads: false`` (``theta_i <- sum_j W_ij theta_j - alpha y_i``, ``y <- W y + g - g_old``) up to rounding.

``s_h`` and ``s_g`` are only valid for a fixed mixing matrix, so the graph must not change during the run, as with
CHOCO-SGD: ``update_graph`` may not be true, and link-drop fault injection or a moving graph plan are refused.  Only the
synchronous (Jacobi) order on undirected graphs exists.
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from .choco import check_static_plan
from ..ops import consensus_ref as ref

FIXED_W = "s_h = sum_j W_ij h_j and s_g = sum_j W_ij g_j are only valid for a fixed W"


class BEER(ConsensusOptimizer):
    alg_name = "beer"
    STATE = ("h", "s_h", "v", "g", "s_g", "m_old", "code_h", "code_g")

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("beer runs the synchronous (jacobi) mixing order only")
        if conf.get("update_graph", False):
            raise ValueError(f"beer needs a fixed graph: {FIXED_W} (update_graph must be false)")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("beer needs a fixed graph: link-drop fault_injection changes it during the run")
        graph = getattr(self.pr, "graph", None)
        if graph is not None and hasattr(graph, "is_directed") and graph.is_directed():
            raise ValueError("beer needs an undirected graph (a doubly stochastic Metropolis matrix)")
        self.alpha = float(conf["alpha"])
        self.gamma = float(conf["gamma"])
        if not 0.0 < self.gamma <= 1.0:
            raise ValueError(f"beer gamma must be in (0, 1] (got {self.gamma})")
        self.compressor = conf["compressor"]
        if self.compressor not in ref.CHOCO_COMPRESSORS:
            raise ValueError(f"beer compressor must be one of {ref.CHOCO_COMPRESSORS} (got {self.compressor!r})")
        self.refresh_graph = False
        a = self.arena
        if a.n_pad % 128 != 0:
            raise ValueError(f"beer needs rows padded to a multiple of 128 elements (n_pad = {a.n_pad})")
        self.live = ref.choco_live(a.layout).to(self.device)
        self.topk_k = ref.choco_k(conf, self.compressor, self.live, "beer")     # entries of a top-k code row (else None)
        self.code_bytes = ref.choco_code_bytes(self.compressor, a.n_pad, a.dtype, self.topk_k)
        self.h, self.s_h = a.zeros(), a.zeros()
        self.v, self.g, self.s_g = a.zeros(), a.zeros(), a.zeros()
        self.m_old = a.zeros()
        # the code rows published at the end of the last round (all zero before round 0: they decode to 0)
        self.code_h = torch.zeros(a.L, self.code_bytes, dtype=torch.uint8, device=self.device)
        self.code_g = torch.zeros_like(self.code_h)

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, 1, 0, refresh=False), "beer", FIXED_W)
            self._plan_checked = True

    def _decode_all(self, code):
        a = self.arena
        return ref.choco_decode(self.pr.gather_rows(code), self.compressor, a.n_pad, a.dtype, self.live, self.topk_k)

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        topo = pr.topology()
        with torch.no_grad():
            ref.beer_mix_(a.theta, self.h, self.s_h, self.v, self.s_g, self._decode_all(self.code_h),
                          self._decode_all(self.code_g), self._rows(topo, topo.W), self.gamma, self.alpha)
        pr.compute_grads()
        with torch.no_grad():
            qh, qg = ref.beer_step_(a.theta, self.h, self.v, self.g, self.s_g, self.m_old, a.grad, self.gamma,
                                    self.compressor, self.live, self.topk_k)
            self.code_h.copy_(qh)
            self.code_g.copy_(qg)
