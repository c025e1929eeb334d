"""SPARQ-SGD — event-triggered compressed gossip with local steps (Singh, Data, George, Diggavi, *SPARQ-SGD:
Event-Triggered and Compressed Communication in Decentralized Optimization*).  No counterpart in the reference.

CHOCO-SGD's memory-efficient compressed gossip (``optimizers/choco.py``), where a node publishes a new code only when
its model has moved far enough from the estimate ``x_hat`` its neighbors hold, and takes ``local_steps`` (H) gradient
steps between communications.  With DSGD's step schedule ``alpha_k`` and the consensus step ``gamma`` in (0, 1],
round k of node i is

    mix:      s_i += sum over j in {i} u N_i with trig_j^{k-1} = 1 of W_ij dec(q_j)   (nothing triggered before round 0)
              theta_i += gamma (s_i - x_hat_i)
    steps:    for p = 0 .. H-1:  theta_i -= alpha_k grad loss_i(theta_i)            (one minibatch draw per step)
    trigger:  e_i = ||theta_i - x_hat_i||^2 (float64);  trig_i^k = e_i > thr_k
    publish:  trig:  q_i = Q(theta_i - x_hat_i);  x_hat_i += dec(q_i);  publish q_i with the tail {1, e_i}
              else:  publish the tail {0, e_i} only (x_hat_i and the code body stay as they are)

The trigger test compares the squared distance to a threshold proportional to ``alpha_k^2``, SPARQ-SGD's form
``c_k alpha_k^2``.  This project picks ``c_k = threshold (k + 1)^threshold_growth`` (``threshold_growth`` in [0, 1),
default 0: a constant ``c``).  ``threshold: 0`` with one local step is CHOCO-SGD bit for bit: a zero difference does not
trigger, and CHOCO would have decoded it to 0.  A threshold above every ``e_i`` never triggers: the run is N
independent SGD runs and pulls no code body.

A published row is the CHOCO code row followed by a 16-byte tail (``ops/consensus_ref.py``); only ``none``, ``int8``
and ``sign`` are available (a top-k row is selected by a cluster kernel that has no trigger).  ``triggers`` counts the
rounds each node triggered in; with the fixed degrees it gives the bytes the mixes pulled exactly
(``pulled_bytes``): each neighbor edge pulls a 16-byte tail every round and a code body once per trigger of its
source.  A problem's results file gets ``sparq_triggers`` (per node, at the end) and ``sparq_pulled_bytes`` (network
total, one entry per evaluation point).

State convention (as CHOCO-SGD's): between rounds ``theta`` holds the value after the steps and before the gossip,
``x_hat`` includes the pending code, ``s`` does not yet include the pending codes; ``code`` is the pending row (body
and tail) and ``triggers`` the counters, both saved with the checkpoint.  ``s`` is only valid for a fixed mixing
matrix: changing graphs, link drops, directed graphs, ``mixing_order: reference`` and Byzantine attackers are refused.
"""
from __future__ import annotations

import math
import numbers

import numpy as np
import torch

from .base import ConsensusOptimizer
from .choco import check_static_plan
from ..ops import consensus_ref as ref

FIXED_W = "s = sum_j W_ij x_hat_j is only valid for a fixed W"


def _real(conf, key, default=None):
    v = conf.get(key, default)
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)) or float(v) < 0.0:
        raise ValueError(f"sparq_sgd {key} must be finite and >= 0 (got {v!r})")
    return float(v)


class SparqSGD(ConsensusOptimizer):
    alg_name = "sparq_sgd"
    STATE = ("x_hat", "s", "code", "triggers")
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("sparq_sgd runs the synchronous (jacobi) mixing order only")
        if conf.get("update_graph", False):
            raise ValueError(f"sparq_sgd needs a fixed graph: {FIXED_W} (update_graph must be false)")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and hasattr(graph, "is_directed") and graph.is_directed():
            raise ValueError("sparq_sgd needs an undirected graph (a doubly stochastic Metropolis matrix)")
        if conf.get("byzantine") is not None:
            raise ValueError("sparq_sgd does not model Byzantine attackers (clipped_gossip and bridge do)")
        pconf = getattr(self.pr, "conf", None) or {}
        if pconf.get("fault_injection"):
            raise ValueError("sparq_sgd needs a fixed graph: link-drop fault_injection changes it during the run")
        self.alph0 = _real(conf, "alpha0")
        self.mu = _real(conf, "mu", 0.0)
        self.threshold = _real(conf, "threshold")
        g = conf.get("threshold_growth", 0.0)
        if isinstance(g, bool) or not isinstance(g, numbers.Real) or not 0.0 <= float(g) < 1.0:
            raise ValueError(f"sparq_sgd threshold_growth must be in [0, 1) (got {g!r})")
        self.threshold_growth = float(g)
        gm = conf.get("gamma")
        if isinstance(gm, bool) or not isinstance(gm, numbers.Real) or not 0.0 < float(gm) <= 1.0:
            raise ValueError(f"sparq_sgd gamma must be in (0, 1] (got {gm!r})")
        self.gamma = float(gm)
        self.compressor = conf.get("compressor")
        if self.compressor == "topk":
            raise ValueError("sparq_sgd compressor topk is not available (the top-k code is selected by a cluster "
                             "kernel that has no trigger); use none, int8 or sign")
        if self.compressor not in ref.SPARQ_COMPRESSORS:
            raise ValueError(f"sparq_sgd compressor must be one of {ref.SPARQ_COMPRESSORS} (got {self.compressor!r})")
        h = conf.get("local_steps", 1)
        if isinstance(h, bool) or not isinstance(h, numbers.Integral) or int(h) < 1:
            raise ValueError(f"sparq_sgd local_steps must be an integer >= 1 (got {h!r})")
        self.local_steps = int(h)
        self.alph = self.alph0
        self.refresh_graph = False
        a = self.arena
        if a.n_pad % 128 != 0:
            raise ValueError(f"sparq_sgd needs rows padded to a multiple of 128 elements (n_pad = {a.n_pad})")
        self.live = ref.choco_live(a.layout).to(self.device)
        self.code_bytes = ref.choco_code_bytes(self.compressor, a.n_pad, a.dtype)
        self.row_bytes = ref.sparq_row_bytes(self.code_bytes)
        self.x_hat = a.zeros()
        self.s = a.zeros()
        # the row published at the end of the last round (all zero before round 0: no trigger)
        self.code = torch.zeros(a.L, self.row_bytes, dtype=torch.uint8, device=self.device)
        self.triggers = torch.zeros(a.L, dtype=torch.int64, device=self.device)
        self._thr = None
        self._pulled = []

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``): DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    def threshold_table(self, n=None) -> np.ndarray:
        """The trigger thresholds of rounds 0..n-1 (default: all ``outer_iterations``), float64."""
        return ref.sparq_threshold(self.threshold, self.threshold_growth, self.alpha_table(n))

    def _before_training(self):
        if not getattr(self, "_plan_checked", False):
            check_static_plan(self.pr.plan_graphs(self.oits, self.k, self.local_steps, 0, refresh=False), "sparq_sgd",
                              FIXED_W)
            self._plan_checked = True

    # -- reports ---------------------------------------------------------------------------------------------------
    def _pending_rows(self) -> torch.Tensor:
        """This rank's rows published for round k (body and tail)."""
        prog = getattr(self, "_program", None)
        if prog is not None and self._use_engine():
            return prog.eng.pub[self.k & 1, 0, :self.pr.placement.L].view(torch.uint8)
        return self.code

    def pulled_bytes(self) -> int:
        """Bytes the mixes of rounds 0 .. k-1 pulled over the whole network: every neighbor edge a 16-byte tail per
        round, and ``code_bytes`` per trigger of its source that a mix has read (the triggers of round k - 1 are read
        by round k's mix)."""
        topo = self.pr.topology()
        deg = torch.as_tensor(np.asarray(topo.deg, dtype=np.int64))
        trig = self.pr.gather_rows(self.triggers).cpu().to(torch.int64)
        pending, _ = ref.sparq_tail_read(self.pr.gather_rows(self._pending_rows()).cpu(), self.code_bytes)
        bodies = int((deg * (trig - pending.to(torch.int64))).sum())
        return ref.SPARQ_TAIL * int(self.k) * int(deg.sum()) + self.code_bytes * bodies

    def choco_bytes(self) -> int:
        """Bytes CHOCO-SGD's mixes of rounds 0 .. k-1 pull: one code row per neighbor edge and round."""
        return self.code_bytes * int(self.k) * int(np.asarray(self.pr.topology().deg).sum())

    def _pulled_list(self) -> list:
        metrics = getattr(self.pr, "metrics", None)
        return metrics.setdefault("sparq_pulled_bytes", []) if isinstance(metrics, dict) else self._pulled

    def _maybe_eval(self, k: int):
        super()._maybe_eval(k)
        if k % self._eval_every() == 0 or k == self.oits - 1:
            self._pulled_list().append(self.pulled_bytes())

    def train(self, profiler=None):
        super().train(profiler)
        trig = self.pr.gather_rows(self.triggers).cpu().to(torch.int64)
        metrics = getattr(self.pr, "metrics", None)
        if isinstance(metrics, dict):
            metrics["sparq_triggers"] = trig
        pulled, choco = self.pulled_bytes(), self.choco_bytes()      # pulled_bytes gathers over the ranks
        if self.pr.ctx.is_main:
            share = pulled / choco if choco else 0.0
            print(f"[nndt] sparq_sgd: {int(trig.sum())} of {int(self.k) * trig.numel()} node-rounds triggered; "
                  f"pulled {pulled} bytes, {100.0 * share:.1f} % of CHOCO-SGD's {choco}", flush=True)

    # -- round -----------------------------------------------------------------------------------------------------
    def _round(self, k: int):
        pr, a = self.pr, self.arena
        topo = pr.topology()
        if self._thr is None:
            self._thr = self.threshold_table()
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            ref.sparq_mix_(a.theta, self.x_hat, self.s, pr.gather_rows(self.code), self._rows(topo, topo.W),
                           self.gamma, self.compressor, self.live, self.code_bytes)
        for _ in range(self.local_steps):
            pr.compute_grads()
            with torch.no_grad():
                ref.sparq_step_(a.theta, a.grad, self.alph)
        with torch.no_grad():
            trig, _ = ref.sparq_publish_(a.theta, self.x_hat, self.code, float(self._thr[k]), self.compressor,
                                         self.live)
            self.triggers.add_(trig.to(torch.int64))
