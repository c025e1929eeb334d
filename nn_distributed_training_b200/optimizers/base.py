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
    def capturable_grads(self) -> bool:
        """True when ``compute_grads`` may be captured in a CUDA graph and replayed: the inner problem's
        ``batched_grads`` hook reads only tensors at fixed addresses and has no per-call host side effects, which the
        problem states with its own ``capturable_grads``.  Otherwise the consensus kernels run eagerly around it."""
        return getattr(self.inner, "batched_grads", None) is not None and bool(getattr(self.inner, "capturable_grads", False))

    def plan_graphs(self, oits: int, k0: int, draws_per_round: int, init_draws: int = 0, refresh: bool = True):
        """Communication graph of rounds ``0..oits-1``: the inner problem's graph, which is static."""
        return [self.inner.graph] * oits

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
        # rounds [0, horizon) whose schedules the fused engine builds (None: all oits); a driver that knows it stops early
        # (the PPO trainers stop at max_rl_timesteps) sets it so no table of outer_iterations entries is built
        self.horizon = None
        self.k = 0  # next round to execute (resume point)
        self.mixing_order = conf.get("mixing_order", "jacobi")
        if self.mixing_order not in ("jacobi", "reference"):
            raise ValueError("mixing_order must be 'jacobi' or 'reference'")
        if self.mixing_order == "reference" and self.pr.ctx.is_distributed:
            raise ValueError("reference (Gauss-Seidel) mixing order is a single-process oracle mode")
        self.checkpointer = None  # set by utils.checkpoint.attach
        if isinstance(self.pr, ConsensusProblem):
            self.pr.privacy_record = None   # a differentially private optimizer sets its own after this
            self.pr.xg_grad_evals = None    # so does the cross-gradient optimizer, with its gradient evaluations

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
            self.fused_program().run(n)
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
        self.fused_program().prepare(n)

    def fused_program(self):
        """The ``RoundProgram`` of the fused consensus kernels, built on first use (DSGT's initial gradient, with
        ``init_grads``, runs then)."""
        prog = getattr(self, "_program", None)
        if prog is None:
            from ..ops.round_program import RoundProgram
            prog = self._program = RoundProgram(self)
            if self.alg_name == "dsgt":
                if self.init_grads and not self._initialised:
                    prog.dsgt_init()
                self._initialised = True
        return prog

    def _use_engine(self) -> bool:
        """Fused sm_90a consensus kernels.  ``consensus_backend``: ``torch`` never; ``auto`` (default) for any arena
        problem on a CUDA device with the synchronous (Jacobi) update order, while foreign problem objects, CPU/gloo and
        the reference-order oracle mode keep the PyTorch ops; ``fused`` also for a foreign problem (through
        ``ReferenceProblemAdapter``), and a configuration the kernels cannot run raises ``ValueError`` naming why."""
        backend = self.conf.get("consensus_backend", "auto")
        if backend == "torch":
            return False
        if backend != "fused" and not isinstance(self.pr, ConsensusProblem):
            return False
        why = self._engine_unsupported()
        if why is not None and backend == "fused":
            raise ValueError(f"consensus backend 'fused' cannot run this {self.alg_name.upper()} run: {why}")
        return why is None

    def _engine_unsupported(self) -> Optional[str]:
        """Why the fused consensus kernels cannot run this optimizer (``None`` if they can)."""
        if self.mixing_order != "jacobi":
            return f"mixing_order {self.mixing_order!r} runs on the PyTorch ops only"
        if self.device.type != "cuda":
            return f"it needs a CUDA device (the device is {self.device})"
        if self.arena.dtype not in (torch.float32, torch.float64):
            return f"parameter dtype {self.arena.dtype} (needs float32 or float64)"
        from ..ops import fused_available
        if not fused_available():
            return "no CUDA device or no sm_90a extension is available"
        return None

    def _round(self, k: int):
        raise NotImplementedError

    def _train_fused(self, profiler):
        from ..ops.round_program import run_fused_training
        run_fused_training(self, profiler)

    # -- checkpoint / resume (SURVEY §5.4: the reference has none) ---------
    # What a checkpoint carries beyond ``k`` and ``theta`` to resume bit-exactly: ``STATE`` names the optimizer's rows
    # of the rank's nodes, ``SCALARS`` its host scalars.  A row that exists only in some configurations is listed only
    # there (an instance sets its own tuple); a listed row that is ``None`` is saved as ``None`` and not restored.
    STATE = ()
    SCALARS = ()

    def state_dict(self) -> Dict:
        sd = {"k": self.k, "theta": self.arena.theta.detach().cpu().clone()}
        sd.update({name: getattr(self, name) for name in self.SCALARS})
        for name in self.STATE:
            row = getattr(self, name)
            sd[name] = None if row is None else row.cpu().clone()
        return sd

    def load_state_dict(self, sd: Dict):
        self.k = int(sd["k"])
        self.arena.theta.copy_(sd["theta"].to(self.device))
        for name in self.SCALARS:       # with the type the attribute has in a freshly built optimizer (float, int)
            setattr(self, name, type(getattr(self, name))(sd[name]))
        for name in self.STATE:
            row = getattr(self, name)
            if row is not None and sd[name] is not None:
                row.copy_(sd[name].to(self.device))
