"""Moniqua — modulo-quantized gossip (Lu, De Sa, *Moniqua: Modulo Quantized Communication in Decentralized SGD*, ICML
2020) on DSGD or on Exact Diffusion (the paper's D² variant).  No counterpart in the reference.

A node publishes ``bits``-bit codes of its parameters taken modulo the range ``B = 2 theta_bound / (1 - 2 delta)``,
``delta = 2^-bits``, with stochastic rounding; a reader decodes them against its own parameters (byte layout and
arithmetic in ``ops/consensus_ref.py``).  While every edge satisfies ``|theta_j - theta_i|_inf <= theta_bound`` the
decoded value ``xhat_j`` is unbiased, within ``B delta`` of ``theta_j`` and the same bits at every reader, so the mix
conserves the network sum.  Nothing depends on the previous round's graph: changing graphs, link drops and the moving
online-density graph are allowed.  With DSGD's step schedule ``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})``, round k of
node i is

    mix:   theta_i += sum_{j != i} w_ij (xhat_j - xhat_i)     (codes published at the end of round k-1; round 0 reads
                                                              the codes of theta^0; w = W, or A = (I + W) / 2 with
                                                              base exact_diffusion; fp64, rounded once)
    step:  DSGD's theta_i -= alpha_k g_i, or Exact Diffusion's adapt / correct (ed_step_, psi <- theta in round 0)
           publish the code of theta_i

State convention (checkpoints and the fused engine rely on it, as CHOCO-SGD's): between rounds ``theta`` holds the value
after the step, the value behind the pending code row ``code``; ``psi`` (Exact Diffusion base) and ``margin``, the
margin hits per node, are state too.

A violated bound decodes silently to the wrong representative.  Two checks report it: ``margin`` counts the neighbor
elements whose decode offset passes ``1/2 - delta`` (the fused mix counts them on the device), and at every evaluation
point the edge gap ``max over the round's edges of |theta_j - theta_i|_inf / theta_bound`` is computed from the true
rows.  A problem's results file gets ``moniqua_margin_hits`` (per node) and ``moniqua_edge_gap`` (one ratio per
evaluation point), and the end of training warns when a hit count is non-zero or a ratio is above 1.  Directed graphs,
``mixing_order: reference`` and Byzantine attackers are refused.
"""
from __future__ import annotations

import math
import numbers

import torch

from .base import ConsensusOptimizer
from ..ops import consensus_ref as ref


def _real(conf, key, default=None, positive=False):
    v = conf.get(key, default)
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)) or float(v) < 0.0 \
            or (positive and float(v) == 0.0):
        raise ValueError(f"moniqua {key} must be finite and {'> 0' if positive else '>= 0'} (got {v!r})")
    return float(v)


class Moniqua(ConsensusOptimizer):
    alg_name = "moniqua"
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("moniqua runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and graph.is_directed():
            raise ValueError("moniqua needs an undirected graph (its mix conserves the network sum only with symmetric "
                             "weights)")
        if conf.get("byzantine") is not None:
            raise ValueError("moniqua does not model Byzantine attackers (clipped_gossip and bridge do)")
        self.alph0 = _real(conf, "alpha0")
        self.mu = _real(conf, "mu", 0.0)
        self.theta_bound = _real(conf, "theta_bound", positive=True)
        bits = conf.get("bits")
        if isinstance(bits, bool) or not isinstance(bits, numbers.Integral) or int(bits) not in ref.MQ_BITS:
            raise ValueError(f"moniqua bits must be one of {ref.MQ_BITS} (got {bits!r})")
        self.bits = int(bits)
        self.base = conf.get("base", "dsgd")
        if self.base not in ref.MQ_BASES:
            raise ValueError(f"moniqua base must be one of {ref.MQ_BASES} (got {self.base!r})")
        seed = conf.get("rounding_seed", getattr(self.pr, "seed", 0))
        if isinstance(seed, bool) or not isinstance(seed, numbers.Integral):
            raise ValueError(f"moniqua rounding_seed must be an integer (got {seed!r})")
        self.rounding_seed = int(seed)
        self.key = ref.mq_key(self.rounding_seed)
        self.B = ref.mq_range(self.theta_bound, self.bits)
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        a, pl = self.arena, self.pr.placement
        self.code_bytes = ref.mq_code_bytes(a.n_pad, self.bits)
        self.live = ref.choco_live(a.layout).to(self.device)
        self.nodes = list(range(pl.lo, pl.lo + pl.L))
        self.psi = a.zeros() if self.base == "exact_diffusion" else None
        self.margin = torch.zeros(pl.L, dtype=torch.int64, device=self.device)
        self.code = torch.zeros(pl.L, self.code_bytes, dtype=torch.uint8, device=self.device)
        self.STATE = ("code", "margin") + (("psi",) if self.psi is not None else ())
        self._gap_due = False
        self._gaps = []
        self.encode_initial()

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def encode_initial(self) -> None:
        """The codes of theta^0, which round 0 reads."""
        with torch.no_grad():
            self.code.copy_(ref.mq_encode(self.arena.theta, self.B, self.bits, self.key, 0, self.nodes, self.live))

    # -- reports ---------------------------------------------------------------------------------------------------
    def _edge_gaps(self) -> list:
        """The edge-gap ratios of the evaluation points so far: the problem's ``moniqua_edge_gap`` metric list (saved
        and restored with the problem's metrics), or the optimizer's own list for a foreign problem."""
        metrics = getattr(self.pr, "metrics", None)
        return metrics.setdefault("moniqua_edge_gap", []) if isinstance(metrics, dict) else self._gaps

    def _record_gap(self, topo) -> None:
        edges = [(i, j) for i in range(topo.W.shape[0]) for j in topo.neighbors_noself[i] if i < j]
        with torch.no_grad():
            rows = self.pr.all_theta() if hasattr(self.pr, "all_theta") else self.pr.gather_rows(self.arena.theta)
            self._edge_gaps().append(ref.mq_edge_gap(rows, edges, self.theta_bound))

    def _maybe_eval(self, k: int):
        super()._maybe_eval(k)
        if k % self._eval_every() == 0 or k == self.oits - 1:
            prog = getattr(self, "_program", None)
            if prog is not None and self._use_engine():     # the planned graph of round k
                self._record_gap(prog.eng.topos[prog.eng.gid[k]])
            else:                                           # recorded in _round(k), after its graph update
                self._gap_due = True

    def margin_hits(self) -> torch.Tensor:
        """Margin hits of every node so far, ``[N]`` int64 on the CPU."""
        return self.pr.gather_rows(self.margin).cpu()

    def train(self, profiler=None):
        super().train(profiler)
        hits = self.margin_hits()
        gaps = self._edge_gaps()
        metrics = getattr(self.pr, "metrics", None)
        if isinstance(metrics, dict):
            metrics["moniqua_margin_hits"] = hits
        worst = max(gaps) if gaps else 0.0
        if (int(hits.sum()) != 0 or worst > 1.0) and self.pr.ctx.is_main:
            print(f"[nndt] WARNING: moniqua left its decode guarantee: {int(hits.sum())} margin hits on "
                  f"{int((hits != 0).sum())} nodes, largest edge gap {worst:.3f} x theta_bound ({self.theta_bound}); "
                  f"raise theta_bound", flush=True)

    # -- round -----------------------------------------------------------------------------------------------------
    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        if k == 0:
            self.encode_initial()
        if self._gap_due:
            self._record_gap(topo)
            self._gap_due = False
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        w = ref.ed_weights(topo.W) if self.psi is not None else topo.W
        with torch.no_grad():
            codes_all = ref.mq_unpack(pr.gather_rows(self.code), self.bits)
            nbrs = [topo.neighbors_noself[g] for g in self.nodes]
            ref.mq_mix_(a.theta, codes_all, self._rows(topo, w), nbrs, self.nodes[0] if self.nodes else 0, self.B,
                        self.bits, self.margin)
        pr.compute_grads()
        with torch.no_grad():
            self.code.copy_(ref.mq_step_(a.theta, self.psi, a.grad, self.alph, k == 0, self.B, self.bits, self.key, k,
                                         self.nodes, self.live))
