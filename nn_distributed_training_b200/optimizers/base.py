"""Common driver for the consensus optimizers.

The reference optimizers (optimizers/{dinno,dsgd,dsgt}.py) are Python loops
over nodes and parameter tensors.  Here an optimizer is pure control flow over
*batched* ops on the flat arena: per round it issues a handful of fused kernels
(or their PyTorch equivalents) covering every local node at once, and — on the
fused backend — whole blocks of rounds are replayed from one CUDA graph with
rho_k / lr_k / alpha_k read from device-side schedules.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from ..parallel.arena import FlatLayout, NodeArena
from ..parallel.context import DistContext, Placement
from ..problems.base import ConsensusProblem
from ..utils.graph_generation import Topology, TopologyCache


class ReferenceProblemAdapter:
    """Wraps any object exposing the reference's problem API
    (``N, graph, models, local_batch_loss(i), evaluate_metrics, update_graph``)
    so the arena-based optimizers can drive it: all nodes are local, the models'
    parameters are re-pointed into arena rows and gradients come from autograd.
    Used for user-defined problems and the PPO problem (rl/dist_ppo.py).  A problem with a non-None
    ``batched_grads(grad_rows)`` computes every node's gradient in one call instead."""

    fused = None
    backend = "torch"

    def __init__(self, pr, device):
        self.inner = pr
        self.N = pr.N
        self.device = torch.device(device)
        self.ctx = DistContext.single(self.device)
        self.placement = Placement(self.N, 1, 0)
        m0 = pr.models[0]
        self.dtype = next(m0.parameters()).dtype
        self.layout = FlatLayout.from_module(m0)
        self.n = self.layout.n
        self.arena = NodeArena(self.layout, self.N, self.device, self.dtype)
        self.models = pr.models
        for i in range(self.N):
            self.arena.attach(i, pr.models[i])
        self.conf = pr.conf
        self._cache = TopologyCache()
        self.last_losses = torch.zeros(self.N, device=self.device, dtype=self.dtype)

    @property
    def graph(self):
        return self.inner.graph

    def topology(self) -> Topology:
        return self._cache.get(self.inner.graph)

    def update_graph(self):
        return self.inner.update_graph()

    def evaluate_metrics(self, at_end=False):
        return self.inner.evaluate_metrics(at_end=at_end)

    def gather_rows(self, t):
        return t

    def compute_grads(self):
        hook = getattr(self.inner, "batched_grads", None)
        if hook is not None:   # one call fills every node's arena.grad row (e.g. DistPPOProblem's update kernels)
            if getattr(self, "_grad_views", None) is None:
                self._grad_views = [self.layout.views(self.arena.grad[i]) for i in range(self.N)]
            torch.sum(hook(self._grad_views), dim=1, out=self.last_losses)
            return self.last_losses
        for i in range(self.N):
            loss = self.inner.local_batch_loss(i)
            grads = torch.autograd.grad(loss, list(self.models[i].parameters()))
            self.arena.set_row_from_grads(i, grads)
            self.last_losses[i] = loss.detach()
        return self.last_losses


def adapt_problem(pr, device):
    return pr if isinstance(pr, ConsensusProblem) else ReferenceProblemAdapter(pr, device)


class ConsensusOptimizer:
    """Shared round loop: evaluation cadence, profiler hook, checkpointing."""

    alg_name = "base"

    def __init__(self, ddl_problem, device, conf):
        self.pr = adapt_problem(ddl_problem, device)
        self.conf = conf
        self.device = torch.device(device)
        self.oits = int(conf["outer_iterations"])
        self.k = 0  # next round to execute (resume point)
        self.mixing_order = conf.get("mixing_order", "jacobi")
        if self.mixing_order not in ("jacobi", "reference"):
            raise ValueError("mixing_order must be 'jacobi' or 'reference'")
        if self.mixing_order == "reference" and self.pr.ctx.is_distributed:
            raise ValueError("reference (Gauss-Seidel) mixing order is a single-process oracle mode")
        self.checkpointer = None  # set by utils.checkpoint.attach

    # -- helpers ---------------------------------------------------------
    @property
    def arena(self) -> NodeArena:
        return self.pr.arena

    def _eval_every(self) -> int:
        return int(self.pr.conf["metrics_config"]["evaluate_frequency"])

    def _maybe_eval(self, k: int):
        if k % self._eval_every() == 0 or k == self.oits - 1:
            self.pr.evaluate_metrics(at_end=(k == self.oits - 1))

    def _rows(self, topo: Topology, mat: np.ndarray) -> torch.Tensor:
        lo, L = self.pr.placement.lo, self.pr.placement.L
        return torch.as_tensor(mat[lo: lo + L], dtype=self.arena.dtype, device=self.device)

    def _deg(self, topo: Topology) -> torch.Tensor:
        lo, L = self.pr.placement.lo, self.pr.placement.L
        return torch.as_tensor(topo.deg[lo: lo + L], dtype=self.arena.dtype, device=self.device)

    # -- template ----------------------------------------------------------
    def train(self, profiler=None):
        if self._use_engine():
            self._train_fused(profiler)
            return
        else:
            self._before_training()
            while self.k < self.oits:
                k = self.k
                self._maybe_eval(k)
                self._round(k)
                self.k = k + 1
                if profiler is not None:
                    profiler.step()
                if self.checkpointer is not None:
                    self.checkpointer.maybe_save(self)
        return

    def _before_training(self):
        pass

    def run_rounds(self, n: int):
        """Advance ``n`` communication rounds with no evaluation in between (the
        stepping API used by benchmarks and custom training loops)."""
        n = min(int(n), self.oits - self.k)
        if n <= 0:
            return
        if self._use_engine():
            from ..ops.round_program import RoundProgram
            prog = getattr(self, "_program", None)
            if prog is None:
                prog = self._program = RoundProgram(self)
                if self.alg_name == "dsgt":
                    if self.init_grads and not self._initialised:
                        prog.dsgt_init()
                    self._initialised = True
            prog.run(n)
            self.k += n
        else:
            self._before_training()
            for _ in range(n):
                self._round(self.k)
                self.k += 1

    def prepare_rounds(self, n: int):
        """Capture (without executing a round) the CUDA graphs that ``run_rounds(n)`` will replay, so that call is graph
        launches only.  No-op on the PyTorch path."""
        n = min(int(n), self.oits - self.k)
        if n <= 0 or not self._use_engine():
            return
        from ..ops.round_program import RoundProgram
        prog = getattr(self, "_program", None)
        if prog is None:
            prog = self._program = RoundProgram(self)
            if self.alg_name == "dsgt":
                if self.init_grads and not self._initialised:
                    prog.dsgt_init()
                self._initialised = True
        prog.prepare(n)

    def _use_engine(self) -> bool:
        """Fused sm_90a consensus kernels: any arena problem on a CUDA device with the
        synchronous (Jacobi) update order; the PyTorch ops remain for CPU/gloo, for
        foreign problem objects and for the reference-order oracle mode."""
        if self.mixing_order != "jacobi" or not isinstance(self.pr, ConsensusProblem):
            return False
        if self.device.type != "cuda" or self.conf.get("consensus_backend", "auto") == "torch":
            return False
        if self.arena.dtype not in (torch.float32, torch.float64):
            return False
        from ..ops import fused_available
        return fused_available()

    def _round(self, k: int):
        raise NotImplementedError

    def _train_fused(self, profiler):
        from ..ops.round_program import run_fused_training
        run_fused_training(self, profiler)

    # -- checkpoint / resume (SURVEY §5.4: the reference has none) ---------
    def state_dict(self) -> Dict:
        return {"k": self.k, "theta": self.arena.theta.detach().cpu().clone()}

    def load_state_dict(self, sd: Dict):
        self.k = int(sd["k"])
        self.arena.theta.copy_(sd["theta"].to(self.device))
