"""CHOCO-SGD — decentralized SGD with compressed gossip (Koloskova, Stich, Jaggi, ICML 2019), in the memory-efficient
form of the paper's appendix.  No counterpart in the reference.

Nodes publish a *code* of the difference between their parameters and their public estimate ``x_hat`` instead of the
parameters themselves (``compressor``: ``none``, ``int8`` with one scale per 32 elements, ``sign``, one bit per
element and one scale per 32, or ``topk``, the ``k = max(1, ceil(topk_ratio n_live))`` entries of largest magnitude
with their indices, ``topk_ratio`` default 0.01; byte layouts in ``ops/consensus_ref.py``).  ``x_hat_i`` is the sum of node i's decoded
codes, known to every neighbor; ``s_i = sum_j W_ij x_hat_j`` (own term included) is kept by node i, so nobody stores
copies of its neighbors' estimates.  With DSGD's step schedule ``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})`` and the
consensus step ``gamma`` in (0, 1], round k of node i is

    mix:   s_i += W_ii dec(q_i) + sum_j W_ij dec(q_j)      (the codes published at the end of round k-1; zero in round 0)
           theta_i += gamma (s_i - x_hat_i)
    step:  theta_i -= alpha_k grad loss_i(theta_i)
           q_i = Q(theta_i - x_hat_i);  x_hat_i += dec(q_i);  publish q_i

State convention (checkpoints and the fused engine rely on it): between rounds, ``theta`` holds the value after the
gradient step and before the gossip, ``x_hat`` already includes the pending code ``q_i`` and ``s`` does not yet include
the pending codes of the node and its neighbors; the pending code row is ``code`` (saved with the checkpoint).  The own
term of ``s`` is added in the mix, from the node's own published row.  With ``compressor: none`` and ``gamma: 1`` the
iterates are DSGD's (``theta <- W theta; theta -= alpha g``) up to rounding, once the first published codes are in:
round 0 has nothing to gossip, so from a common starting row the two agree from the start.

``s`` is only valid for a fixed mixing matrix, so the graph must not change during the run: ``update_graph`` defaults to
false and may not be true, and a problem whose graph sequence has more than one topology (link-drop fault injection,
a moving online-density plan) is refused.  Only the synchronous (Jacobi) order exists.
"""
from __future__ import annotations

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


class ChocoSGD(ConsensusOptimizer):
    alg_name = "choco_sgd"
    STATE = ("x_hat", "s", "code")
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("choco_sgd runs the synchronous (jacobi) mixing order only")
        if conf.get("update_graph", False):
            raise ValueError("choco_sgd needs a fixed graph: its sum s = sum_j W_ij x_hat_j is only valid for a fixed W "
                             "(update_graph must be false)")
        super().__init__(ddl_problem, device, conf)
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("choco_sgd needs a fixed graph: link-drop fault_injection changes it during the run")
        self.alph0 = float(conf["alpha0"])
        self.mu = float(conf.get("mu", 0.0))
        self.alph = self.alph0
        self.gamma = float(conf["gamma"])
        if not 0.0 < self.gamma <= 1.0:
            raise ValueError(f"choco_sgd gamma must be in (0, 1] (got {self.gamma})")
        self.compressor = conf["compressor"]
        if self.compressor not in ref.CHOCO_COMPRESSORS:
            raise ValueError(f"choco_sgd compressor must be one of {ref.CHOCO_COMPRESSORS} (got {self.compressor!r})")
        self.refresh_graph = False
        a = self.arena
        if a.n_pad % 128 != 0:
            raise ValueError(f"choco_sgd needs rows padded to a multiple of 128 elements (n_pad = {a.n_pad})")
        self.live = ref.choco_live(a.layout).to(self.device)
        self.topk_k = ref.choco_k(conf, self.compressor, self.live, "choco_sgd")     # entries of a top-k code row (else None)
        self.code_bytes = ref.choco_code_bytes(self.compressor, a.n_pad, a.dtype, self.topk_k)
        self.x_hat = a.zeros()
        self.s = a.zeros()
        # the code row published at the end of the last round (all zero before round 0: it decodes to 0)
        self.code = torch.zeros(a.L, self.code_bytes, dtype=torch.uint8, device=self.device)

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, 1, 0, refresh=False))
            self._plan_checked = True

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        topo = pr.topology()
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            dec_all = ref.choco_decode(pr.gather_rows(self.code), self.compressor, a.n_pad, a.dtype, self.live,
                                       self.topk_k)
            ref.choco_mix_(a.theta, self.x_hat, self.s, dec_all, self._rows(topo, topo.W), self.gamma)
        pr.compute_grads()
        with torch.no_grad():
            self.code.copy_(ref.choco_step_(a.theta, self.x_hat, a.grad, self.alph, self.compressor, self.live,
                                            self.topk_k))


def check_static_plan(graphs, alg="choco_sgd", why="s = sum_j W_ij x_hat_j is only valid for a fixed W"):
    """Raise ``ValueError`` when a planned graph sequence holds more than one topology (``alg`` and ``why`` name the
    optimizer and its reason in the message)."""
    from ..utils.graph_generation import Topology
    keys = set()
    seen = set()
    for g in graphs:
        if id(g) in seen:
            continue
        seen.add(id(g))
        keys.add(Topology(g).key)
        if len(keys) > 1:
            raise ValueError(f"{alg} needs a fixed graph: the planned graph sequence of this problem changes "
                             f"during the run ({why})")
