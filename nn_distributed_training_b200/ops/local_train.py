"""Fused training of nodes that do not communicate: the solo ("individual") and centralized baselines.

The nodes are built as an existing problem on an edgeless graph, so ``FusedMnist`` / ``FusedMLP`` train and evaluate
them unchanged.  A step is [forward/backward of every node, ``local_step``]: the step kernel (csrc/consensus.cu:
local_step_kernel) sums each node's gradient partials and applies one torch.optim SGD / Adam / AdamW step while the
node's step counter is below its budget of ``epochs x batches_per_epoch`` steps.  A node with a smaller shard reaches
its budget earlier and is left untouched from then on.  ``max(budget)`` steps run as CUDA graphs of up to
``STEPS_PER_GRAPH`` steps (``NNDT_NO_GRAPH=1``: eager launches), with no host work per step.

Batches come from the in-kernel Feistel sampler (``data.sampler.BatchSchedule`` is its host twin), not from
``torch.randperm``: a run is a different draw of the same experiment than the torch path.
"""
from __future__ import annotations

import gc
import os
from typing import Dict, List, Sequence

import networkx as nx
import torch

from . import load_ext, mlp_kernel_supports, mnist_kernel_supports
from ..data.sampler import BatchSchedule
from ..data.shards import as_shard
from ..parallel.context import DistContext
from .engine import OPT_CODE

STEPS_PER_GRAPH = 64
SOLO_OPTIMIZERS = ("sgd", "adam", "adamw")
BACKENDS = ("torch", "fused")


def epoch_budgets(sizes: Sequence[int], batch: int, epochs: int) -> List[int]:
    """Steps each node takes: ``epochs`` DataLoader epochs of its shard, the partial last batch included."""
    return [int(epochs) * BatchSchedule(int(m), int(batch)).batches_per_epoch for m in sizes]


def check_fused(kind: str, model, loss, device, batch: int, optimizer: str) -> None:
    """Raise ``ValueError`` naming why the fused baseline cannot run ``model`` / ``loss`` / ``optimizer`` on ``device``
    (``kind``: mnist | density)."""
    device = torch.device(device)
    if device.type != "cuda" or not torch.cuda.is_available():
        raise ValueError(f"individual_training.backend: fused needs a CUDA device (got {device})")
    if load_ext() is None:
        raise ValueError("individual_training.backend: fused needs the sm_90a extension, which is not built")
    if optimizer not in SOLO_OPTIMIZERS:
        raise ValueError(f"individual_training.backend: fused runs {'/'.join(SOLO_OPTIMIZERS)}, not {optimizer!r}")
    spec = getattr(model, "spec", None)
    dtype = next(model.parameters()).dtype
    if kind == "mnist":
        from ..models.spec import ConvNetSpec
        ok = (isinstance(spec, ConvNetSpec) and isinstance(loss, torch.nn.NLLLoss)
              and mnist_kernel_supports(spec, int(batch), dtype))
    else:
        from ..models.spec import MLPSpec
        ok = isinstance(spec, MLPSpec) and mlp_kernel_supports(spec, loss, dtype)
    if not ok:
        raise ValueError(f"individual_training.backend: fused has no kernel for {type(model).__name__} "
                         f"(spec={spec}, loss={type(loss).__name__}, dtype={dtype}, batch={batch})")


def build_problem(kind: str, model, loss, shards, val, device, batch: int, val_batch: int, seed: int):
    """Every shard as one node of an edgeless graph, on the fused backend of this process's device."""
    from ..problems import DistDensityProblem, DistMNISTProblem
    cls = DistMNISTProblem if kind == "mnist" else DistDensityProblem
    conf = dict(problem_name="local", train_batch_size=int(batch), val_batch_size=int(val_batch), metrics=[])
    dev = torch.device(device)
    return cls(nx.empty_graph(len(shards)), model, loss, [as_shard(s) for s in shards], val, dev, conf,
               ctx=DistContext.single(dev), backend="fused", seed=int(seed))


class LocalTrainer:
    """Owns the optimizer state, step counters and captured graphs of one fused local-training run."""

    def __init__(self, problem, optimizer: str, lr: float, budgets: Sequence[int]):
        if optimizer not in SOLO_OPTIMIZERS:
            raise ValueError(f"no fused local step for optimizer {optimizer!r}")
        pr = self.pr = problem
        fz = pr.fused
        if fz is None:
            raise ValueError("local training needs a problem on the fused backend")
        a, dev, L = pr.arena, pr.device, pr.placement.L
        if len(budgets) != L:
            raise ValueError(f"{len(budgets)} budgets for {L} nodes")
        self.budget = torch.tensor([int(b) for b in budgets], dtype=torch.int32, device=dev)
        self.total = max(int(b) for b in budgets)
        # the MNIST kernels advance their own draw counters; the step kernel then counts steps in a counter of its own
        self.steps = (torch.zeros(L, dtype=torch.int32, device=dev) if getattr(fz, "owns_calls", False) else fz.calls)
        self.arrive = torch.zeros(L, dtype=torch.int32, device=dev)
        adam = optimizer != "sgd"
        self.m = torch.zeros_like(a.theta) if adam else None
        self.v = torch.zeros_like(a.theta) if adam else None
        d = dict(L=L, n_pad=a.n_pad, S=fz.S, theta=a.theta.data_ptr(), grad_part=fz.grad_part.data_ptr(),
                 calls=self.steps.data_ptr(), budget=self.budget.data_ptr(), arrive=self.arrive.data_ptr(),
                 m=self.m.data_ptr() if adam else None, v=self.v.data_ptr() if adam else None,
                 local_lr=float(lr), opt=OPT_CODE[optimizer])
        ext = load_ext(required=True)
        self.op = (ext.LocalStepOpF32 if a.dtype == torch.float32 else ext.LocalStepOpF64)(d)
        self.capturable = os.environ.get("NNDT_NO_GRAPH", "0") != "1"
        self._graphs: Dict[int, torch.cuda.CUDAGraph] = {}

    def _step(self):
        self.pr.fused.launch()
        self.op.step()

    def _graph(self, r: int) -> torch.cuda.CUDAGraph:
        g = self._graphs.get(r)
        if g is None:
            gc.collect()      # an unreachable earlier run may own graphs; collecting one mid-capture breaks the capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(r):
                    self._step()
            self._graphs[r] = g
        return g

    def run(self, steps: int):
        """Enqueue ``steps`` steps of every node (nodes past their budget stay as they are)."""
        left = int(steps)
        while left > 0:
            r = min(left, STEPS_PER_GRAPH)
            if self.capturable:
                self._graph(r).replay()
            else:
                for _ in range(r):
                    self._step()
            left -= r

    def steps_taken(self) -> List[int]:
        return [int(s) for s in self.steps.cpu()]


def _mnist_eval(pr, val_batch: int):
    """(sum of ``val_batch`` batch-mean losses [L], correct counts [L]) of every node, on the device."""
    from ..problems.base import sum_of_batch_means
    ps, ok = pr.fused.validate()
    return sum_of_batch_means(ps, int(val_batch)), ok.sum(1)


def solo_mnist(model, loss, train_sets, val_set, device, conf, seed: int = 0) -> Dict[int, dict]:
    """Fused twin of ``dist_mnist_ex.train_solo`` for every node at once: ``{node: {validation_loss,
    validation_accuracy}}`` with the torch path's normalisation (sum of batch means / |val|)."""
    bs, vb = int(conf["train_batch_size"]), int(conf["val_batch_size"])
    check_fused("mnist", model, loss, device, bs, conf["optimizer"])
    pr = build_problem("mnist", model, loss, train_sets, val_set, device, bs, vb, seed)
    tr = LocalTrainer(pr, conf["optimizer"], conf["lr"], epoch_budgets(pr.node_sizes, bs, conf["epochs"]))
    tr.run(tr.total)
    vl, corr = _mnist_eval(pr, vb)
    V = len(pr.val)
    vl, corr = vl.cpu(), corr.cpu()
    return {g: {"validation_loss": float(vl[g]) / V, "validation_accuracy": int(corr[g]) / V} for g in range(pr.N)}


def solo_density(model, loss, train_sets, val_set, device, conf, seed: int = 0) -> Dict[int, dict]:
    """Fused twin of ``density_common.train_solo`` for every node at once.  A node trains on epochs of its whole
    trajectory shard (the offline problem: no sliding window).  Returns ``{node: {validation_loss,
    mesh_grid_density, mesh_grid}}`` as CPU tensors."""
    from ..experiments.density_common import mesh_inputs
    bs, vb = int(conf["train_batch_size"]), int(conf["val_batch_size"])
    check_fused("density", model, loss, device, bs, conf["optimizer"])
    shards = [as_shard(s) for s in train_sets]
    pr = build_problem("density", model, loss, shards, val_set, device, bs, vb, seed)
    tr = LocalTrainer(pr, conf["optimizer"], conf["lr"], epoch_budgets(pr.node_sizes, bs, conf["epochs"]))
    tr.run(tr.total)
    vl = pr._val_losses_local().cpu()
    mesh = mesh_inputs(val_set, pr.device, pr.dtype)
    dense = pr._forward_local(mesh).cpu()
    mesh = mesh.cpu()
    return {g: {"validation_loss": vl[g].clone(), "mesh_grid_density": dense[g].reshape(-1, 1).clone(),
                "mesh_grid": mesh.clone()} for g in range(pr.N)}


def centralized(model, loss, train, val, device, epochs: int, lr: float, batch: int, val_batch: int,
                squeeze: bool, verbose: bool = True, seed: int = 0) -> List[dict]:
    """Fused twin of ``centralized.train_centralized``: one node on the union shard, Adam, evaluated after every epoch
    into the same ``hist`` records."""
    kind = "density" if squeeze else "mnist"
    check_fused(kind, model, loss, device, batch, "adam")
    pr = build_problem(kind, model, loss, [train], val, device, batch, val_batch, seed)
    bpe = BatchSchedule(int(pr.node_sizes[0]), int(batch)).batches_per_epoch
    tr = LocalTrainer(pr, "adam", lr, [int(epochs) * bpe])
    hist = []
    for ep in range(int(epochs)):
        tr.run(bpe)
        if squeeze:
            rec = {"epoch": ep, "validation_loss": float(pr._val_losses_local()[0]), "top1_accuracy": None}
        else:
            vl, corr = _mnist_eval(pr, val_batch)
            rec = {"epoch": ep, "validation_loss": float(vl[0]), "top1_accuracy": int(corr[0]) / len(pr.val)}
        hist.append(rec)
        if verbose:
            print(rec)
    return hist
