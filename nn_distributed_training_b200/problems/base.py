"""Shared machinery of the distributed-learning problems.

A *problem* owns, for the graph nodes hosted by this rank: the flat parameter
arena and the ``nn.Module`` shells viewing it, the device-resident data shards
with their stateless samplers, and the metric bookkeeping.  It exposes

* the reference's problem API (``N, n, graph, models, conf, metrics, device``,
  ``local_batch_loss(i)``, ``evaluate_metrics(at_end)``, ``update_graph()``,
  ``save_metrics(dir)``, ``validate(i)`` — problems/dist_mnist_problem.py:15-211),
* the batched API the consensus optimizers drive: ``compute_grads()`` fills
  ``arena.grad`` for every local node in one call — a fused sm_90a kernel when
  ``backend == "fused"``, autograd otherwise.
"""
from __future__ import annotations

import copy
import os
from typing import Callable, Dict, List, Optional, Sequence

import networkx as nx
import numpy as np
import torch

from ..data.sampler import BatchSchedule
from ..data.shards import Shard, ShardSet, as_shard
from ..ops import consensus_ref
from ..parallel.arena import FlatLayout, NodeArena
from ..parallel.context import DistContext, Placement
from ..utils.graph_generation import Topology, TopologyCache


def per_sample_loss(base_loss):
    """A ``reduction='none'`` twin of a torch.nn loss module (None if impossible)."""
    if getattr(base_loss, "reduction", None) == "mean":
        twin = copy.copy(base_loss)
        twin.reduction = "none"
        return twin
    return None


def sum_of_batch_means(ps: torch.Tensor, batch: int) -> torch.Tensor:
    """``sum_b mean(ps[b*batch:(b+1)*batch])`` along the last dim — what a
    DataLoader loop that adds ``loss(...).item()`` per batch accumulates
    (problems/dist_mnist_problem.py:122-125)."""
    v = ps.shape[-1]
    full = v // batch
    out = ps.new_zeros(ps.shape[:-1])
    if full:
        out = out + ps[..., : full * batch].reshape(*ps.shape[:-1], full, batch).mean(-1).sum(-1)
    if v - full * batch:
        out = out + ps[..., full * batch:].mean(-1)
    return out


class ConsensusProblem:
    """Base class; subclasses provide data handling, validation and metrics."""

    #: squeeze model output before the loss (density problems)
    squeeze_output = False
    #: ``() -> dict`` of the optimizer training this problem when it is differentially private (optimizers/dp_dsgd.py),
    #: written into the results file as ``privacy``; every optimizer resets it to None when it is built
    privacy_record: Optional[Callable[[], dict]] = None

    def __init__(self, graph, base_model, base_loss, train_sets, val_set, device, conf,
                 ctx: Optional[DistContext] = None, backend: Optional[str] = None,
                 seed: Optional[int] = None):
        self.conf = conf
        self.base_loss = base_loss
        self.base_model = base_model
        self.device = torch.device(device)
        self.ctx = ctx or DistContext.single(self.device)
        self.seed = int(conf.get("seed", 0) if seed is None else seed)

        self._topo_cache = TopologyCache()
        self.train_sets = train_sets
        self.val_set = val_set
        self.N = len(train_sets) if graph is None else graph.number_of_nodes()
        self.placement = Placement(self.N, self.ctx.world_size, self.ctx.rank)
        self.graph = graph
        self._init_faults()

        # ---- parameters: one arena row per local node --------------------
        p0 = next(base_model.parameters())
        self.dtype = p0.dtype
        self.layout = FlatLayout.from_module(base_model)
        self.n = self.layout.n
        self.arena = NodeArena(self.layout, self.placement.L, self.device, self.dtype)
        self.models: Dict[int, torch.nn.Module] = {}
        for l, g in enumerate(self.placement.local_nodes):
            model = copy.deepcopy(base_model).to(self.device)
            self.arena.attach(l, model)
            self.models[g] = model

        # ---- data ---------------------------------------------------------
        self.train_batch_size = int(conf["train_batch_size"])
        self.val_batch_size = int(conf["val_batch_size"])
        self._setup_data(train_sets, val_set)

        # ---- metrics ------------------------------------------------------
        self.metrics = {name: [] for name in conf["metrics"]}
        self.calls = np.zeros(self.N, dtype=np.int64)  # draws per node (all ranks mirror all nodes)
        self.forward_cnt = 0
        self.last_losses = torch.zeros(self.placement.L, device=self.device, dtype=self.dtype)

        # ---- execution backend --------------------------------------------
        self.backend = self._select_backend(backend or conf.get("backend", "auto"))
        self.fused = None
        if self.backend == "fused":
            self._setup_fused()

    # ------------------------------------------------------------------
    # data
    # ------------------------------------------------------------------
    def _setup_data(self, train_sets, val_set):
        shards = [as_shard(train_sets[g]) for g in self.placement.local_nodes]
        self.node_sizes = np.asarray([_len_only(s) for s in train_sets], dtype=np.int64)
        self.shards = ShardSet(shards, self.device)
        self.schedules = [BatchSchedule(int(m), self.train_batch_size) for m in self.node_sizes]
        self.val = as_shard(val_set).to(self.device) if val_set is not None else None

    @property
    def epoch_tracker(self) -> torch.Tensor:
        """Per-node count of DataLoader re-arms, as the reference tracks it."""
        return torch.tensor([self.schedules[g].epochs_completed(int(self.calls[g])) for g in range(self.N)],
                            dtype=torch.get_default_dtype())

    def _draw_indices(self, g: int) -> torch.Tensor:
        """Row indices (into the node's shard) of node ``g``'s next minibatch."""
        idx = self.schedules[g].indices(int(self.calls[g]), self.seed, g, device=self.device)
        self._count_draw(g)
        return idx

    def _count_draw(self, g: int, times: int = 1):
        self.calls[g] += times
        if g == 0:
            # node 0 is the forward-pass odometer (dist_mnist_problem.py:90-94)
            self.forward_cnt += times * self.train_batch_size

    def count_draws_all(self, times: int = 1):
        """Advance the draw counters of *every* node (all nodes draw in lockstep;
        each rank mirrors the whole network so epoch/forward-count metrics and the
        dynamic-graph schedule need no communication)."""
        self.calls += times
        self.forward_cnt += times * self.train_batch_size

    def plan_graphs(self, oits: int, k0: int, draws_per_round: int, init_draws: int = 0, refresh: bool = True):
        """Communication graph of every round ``0..oits-1`` (static here).  Problems
        with a data-driven graph override this; it is what lets a dynamic topology
        live in device tables indexed by the round counter."""
        if self._faults is None:
            return [self.graph] * oits
        return [self.faulted_graph(self._base_graph, k) if refresh else self._base_graph for k in range(oits)]

    def _batch(self, g: int):
        l = self.placement.local_index(g)
        shard = self.shards.shard(l)
        idx = self._draw_indices(g)
        return shard.inputs(idx, self.dtype), shard.targets(idx)

    # ------------------------------------------------------------------
    # losses / gradients
    # ------------------------------------------------------------------
    def _loss(self, model, x, y):
        yh = model(x)
        if self.squeeze_output:
            yh = torch.squeeze(yh)
            y = y.to(yh.dtype)
        return self.base_loss(yh, y)

    def local_batch_loss(self, i: int) -> torch.Tensor:
        """Loss (with autograd graph) of node ``i``'s model on its next batch."""
        x, y = self._batch(i)
        loss = self._loss(self.models[i], x, y)
        self._after_loss(i, loss)
        return loss

    def _after_loss(self, i: int, loss: torch.Tensor):
        pass

    def compute_grads(self) -> torch.Tensor:
        """Next-batch loss and gradient for every local node -> ``arena.grad``;
        returns the ``[L]`` loss vector (device)."""
        if self.fused is not None:
            return self.fused.compute_grads()
        for l, g in enumerate(self.placement.local_nodes):
            loss = self.local_batch_loss(g)
            grads = torch.autograd.grad(loss, list(self.models[g].parameters()))
            self.arena.set_row_from_grads(l, grads)
            self.last_losses[l] = loss.detach()
        for g in range(self.N):  # mirror the lockstep draws of nodes hosted elsewhere
            if not self.placement.is_local(g):
                self._count_draw(g)
        return self.last_losses

    def compute_grads_pair(self, theta_prev: torch.Tensor, grad_prev: torch.Tensor) -> torch.Tensor:
        """``compute_grads`` plus the gradient at a second point on the *same* minibatch: ``arena.grad`` at theta and
        ``grad_prev`` at ``theta_prev`` (both ``[L, n_pad]``).  One draw per node: the draw counters, ``forward_cnt``
        and the losses (of the current point) advance once, as for ``compute_grads``.  Returns the ``[L]`` losses at
        theta."""
        if self.fused is not None:
            return self.fused.compute_grads_pair(theta_prev, grad_prev)
        return self.compute_grads_multi(theta_prev.unsqueeze(0), grad_prev.unsqueeze(0))

    def compute_grads_multi(self, points: torch.Tensor, grads: torch.Tensor) -> torch.Tensor:
        """``compute_grads`` plus the gradient at ``P`` more points on the *same* minibatch: ``arena.grad`` at theta and
        ``grads[p]`` at ``points[p]`` (both ``[P, L, n_pad]``).  One draw per node: the draw counters, ``forward_cnt``
        and the losses (of theta) advance once, as for ``compute_grads``.  On the fused kernels the points are the
        buffers the extra training ops were built on (``enable_cross_points``).  Returns the ``[L]`` losses at theta."""
        if self.fused is not None:
            return self.fused.compute_grads_multi(points, grads)
        for l, g in enumerate(self.placement.local_nodes):
            model = self.models[g]
            x, y = self._batch(g)
            loss = self._loss(model, x, y)
            self._after_loss(g, loss)
            self.arena.set_row_from_grads(l, torch.autograd.grad(loss, list(model.parameters())))
            self.last_losses[l] = loss.detach()
            # the same network at each point on the same batch: leaves viewing the row, through functional_call; the
            # loss hook (_after_loss) sees theta only
            for p in range(points.shape[0]):
                prev = [t.detach().requires_grad_(True) for t in self.layout.views(points[p, l])]
                params = {s.name: t for s, t in zip(self.layout.slots, prev)}

                def at_prev(inp, model=model, params=params):
                    return torch.func.functional_call(model, params, (inp,))
                at_prev.parameters = lambda prev=prev: iter(prev)     # what a loss hook may inspect on a NaN
                loss_p = self._loss(at_prev, x, y)
                for dst, t in zip(self.layout.views(grads[p, l]), torch.autograd.grad(loss_p, prev)):
                    dst.copy_(t)
        for g in range(self.N):
            if not self.placement.is_local(g):
                self._count_draw(g)
        return self.last_losses

    # ------------------------------------------------------------------
    # graph
    # ------------------------------------------------------------------
    def update_graph(self):
        """Static graph: nothing to do (dist_mnist_problem.py:100-102) — unless link-drop fault
        injection is configured, in which case round ``r`` uses the faulted graph."""
        if self._faults is not None:
            self.graph = self.faulted_graph(self._base_graph, self._graph_round)
            self._graph_round += 1
        return

    # ---- fault injection (SURVEY §5.3: the reference has none) ---------------------------
    def _init_faults(self):
        """``fault_injection: {link_drop_prob: p, seed: s, from_round: a, to_round: b}`` in the
        problem config drops every edge independently with probability ``p`` in rounds
        ``[a, b)`` — the same mechanism as a time-varying graph, so it runs on the fused path
        through the planned topology tables.  Nodes left without neighbors take local steps."""
        f = self.conf.get("fault_injection")
        self._faults = dict(f) if f else None
        self._graph_round = 0
        self._base_graph = self.graph

    def faulted_graph(self, graph, rnd: int):
        f = self._faults
        if f is None or graph is None or not (f.get("from_round", 0) <= rnd < f.get("to_round", 10 ** 12)):
            return graph
        rng = np.random.default_rng([int(f.get("seed", 0)), int(rnd)])
        g = graph.copy()
        edges = sorted(tuple(sorted(e)) for e in graph.edges() if e[0] != e[1])
        drop = rng.random(len(edges)) < float(f["link_drop_prob"])
        g.remove_edges_from([e for e, d in zip(edges, drop) if d])
        return g

    def topology(self) -> Topology:
        return self._topo_cache.get(self.graph)

    # ------------------------------------------------------------------
    # gathered views
    # ------------------------------------------------------------------
    def gather_rows(self, local: torch.Tensor) -> torch.Tensor:
        """``[L, ...] -> [N, ...]`` across ranks (identity when single process)."""
        return self.ctx.all_gather_cat(local, self.placement.counts)

    def all_theta(self) -> torch.Tensor:
        return self.arena.compact(self.gather_rows(self.arena.theta))

    # ------------------------------------------------------------------
    # metrics
    # ------------------------------------------------------------------
    def _consensus_metric(self):
        eng = getattr(self, "_metric_engine", None)
        if eng is not None:     # fused path: P2P pull of every node's published row, fp64 accumulation
            d_all, d_mean = eng[0].consensus_metric(eng[1]())
            return d_all.to(torch.get_default_dtype()), d_mean.to(torch.get_default_dtype())
        with torch.no_grad():
            d_all, d_mean = consensus_ref.consensus_error(self.all_theta())
        return d_all, d_mean

    def save_metrics(self, output_dir):
        """``<problem_name>_results.pt`` (dist_mnist_problem.py:104-109); rank 0 only."""
        if not self.ctx.is_main:
            return
        path = os.path.join(output_dir, self.conf["problem_name"] + "_results.pt")
        out = dict(self.metrics)
        if getattr(self, "data_source", None) is not None:
            out["data_source"] = self.data_source     # extra key next to the reference's metric lists
        byz = self.conf.get("optimizer_config", {}).get("byzantine")
        if byz:
            out["byzantine_nodes"] = sorted(int(v) for v in byz["nodes"])   # summaries average the other nodes
        if self.privacy_record is not None:
            out["privacy"] = self.privacy_record()
        if getattr(self, "xg_grad_evals", None) is not None:
            out["xg_grad_evals"] = self.xg_grad_evals
        torch.save(out, path)

    def state_dicts(self) -> Dict[int, dict]:
        """``{node: state_dict}`` for every node (gathered to all ranks)."""
        th = self.gather_rows(self.arena.theta).cpu()
        out = {}
        for g in range(self.N):
            sd = {}
            for slot in self.layout.slots:
                sd[slot.name] = th[g, slot.offset: slot.offset + slot.numel].view(slot.shape).clone()
            out[g] = sd
        return out

    # ------------------------------------------------------------------
    # backend
    # ------------------------------------------------------------------
    def _fused_supported(self) -> bool:
        return False

    def _select_backend(self, want: str) -> str:
        if want not in ("auto", "torch", "fused"):
            raise ValueError(f"unknown backend {want!r}")
        if want == "torch":
            return "torch"
        ok = self.device.type == "cuda" and self.dtype in (torch.float32, torch.float64) and self._fused_supported()
        if want == "fused" and not ok:
            raise RuntimeError("fused sm_90a backend requested but unsupported for this "
                               "device/dtype/model (needs CUDA and a kernel-backed model spec / dtype)")
        if not ok and self.device.type == "cuda" and self.ctx.is_main:
            # never a silent fallback on a GPU box: say which model runs autograd + library kernels and why
            print(f"[nndt] WARNING: no fused forward/backward kernel for {type(self.base_model).__name__} "
                  f"(spec={getattr(self.base_model, 'spec', None)}, dtype={self.dtype}, loss={type(self.base_loss).__name__}): "
                  "forward/backward falls back to PyTorch autograd (cuDNN/cuBLAS); the consensus kernels stay fused",
                  flush=True)
        return "fused" if ok else "torch"

    def _setup_fused(self):  # pragma: no cover - overridden
        raise NotImplementedError


def _len_only(ds) -> int:
    try:
        return len(ds)
    except TypeError:  # pragma: no cover
        return len(as_shard(ds))
