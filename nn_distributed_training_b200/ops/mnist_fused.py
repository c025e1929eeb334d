"""Python side of the fused MNIST kernels (csrc/mnist.cu).

``FusedMnist`` owns the device buffers the kernels read/write for one problem
instance: the flattened uint8/float shard rows, the device draw counters of the
stateless sampler, the per-slice gradient partials and the validation outputs.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import load_ext, mnist_kernel_is_paper_shape

SPB = 8  # samples per CTA of the evaluation kernel / upper bound for training (template instantiations in mnist.cu)


def choose_spb(batch: int, n_local: int, sms: int) -> int:
    """Samples per training CTA (4..8).  A node's batch is cut into ceil(batch/spb) CTAs; per-CTA time grows
    with spb (conv / fc work) on top of a fixed part (weight staging, dW1 write-out), so the best choice is
    the smallest spb whose L x S CTAs still fit in ONE wave of the SMs (1 CTA/SM: ~200 KB smem, 768 threads)."""
    for spb in range(4, SPB + 1):
        if n_local * -(-batch // spb) <= sms:
            return spb
    return SPB


class FusedMnist:
    def __init__(self, problem):
        self.pr = problem
        self.ext = load_ext(required=True)
        dev = problem.device
        a, pl = problem.arena, problem.placement
        self.L, self.n_pad = pl.L, a.n_pad
        self.B = problem.train_batch_size
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        spec = problem.base_model.spec
        self.dtype = a.dtype
        # the paper's (3, 5, 64) net in fp32 runs the specialised kernels; every other shape and all of fp64 run the
        # generic CUDA-core kernel (csrc/mnist_generic.cu)
        self.generic = not (self.dtype == torch.float32 and mnist_kernel_is_paper_shape(spec)) \
            or os.environ.get("NNDT_MNIST_GENERIC") == "1"
        if self.generic:
            d64 = int(self.dtype == torch.float64)
            fits8 = self.ext.convnet_generic_smem_bytes(spec.num_filters, spec.kernel_size, spec.linear_width, d64, 8) <= 200 * 1024
            want = int(os.environ.get("NNDT_GENERIC_SPB", "0")) or (8 if fits8 and self.L * -(-self.B // 8) >= sms // 2 else 4)
            self.spb = 8 if (want == 8 and fits8) else 4
        else:
            self.spb = (int(os.environ.get("NNDT_SPB", "0")) or int(problem.conf.get("samples_per_cta", 0))
                        or choose_spb(self.B, self.L, sms))
            assert 4 <= self.spb <= SPB
        self.S = -(-self.B // self.spb)
        # paper shape, fp32, batch <= 64: the K-split cluster kernel (csrc/mnist_tc.cu) — one gradient
        # row per node instead of S per-slice partials.  NNDT_MNIST_TC=0 keeps the batch-split mma.sync kernel (A/B).
        self.tc = (not self.generic and self.B <= 64 and os.environ.get("NNDT_MNIST_TC", "1") != "0"
                   and str(problem.conf.get("mnist_kernel", "tc")) == "tc" and self.ext.mnist_tc_max_clusters() >= 1)
        if self.tc:
            # batch splits per node (1, 2 or 4 clusters of 6 CTAs, M = 64 / 32 / 16 samples each): as many as keep all
            # 6 * nsplit * L CTAs in one wave — the conv / conv-grad phases are CUDA-core work that scales with SMs
            want = int(os.environ.get("NNDT_TC_SPLIT", "0"))
            self.S = want if want in (1, 2, 4) else max([n for n in (1, 2, 4) if 6 * n * self.L <= sms] or [1])
        # float64, paper shape, batch <= 64: a K-split cluster kernel with the fc1 contractions on the FP64 tensor cores
        # (csrc/mnist_cl64.cu); NNDT_MNIST_CL64=0 keeps the batch-split generic kernel (A/B)
        self.cl64 = (self.generic and self.dtype == torch.float64 and mnist_kernel_is_paper_shape(spec) and self.B <= 64
                     and os.environ.get("NNDT_MNIST_CL64", "1") != "0")
        if self.cl64:
            want = int(os.environ.get("NNDT_TC_SPLIT", "0"))
            split = want if want in (1, 2, 4) else max([n for n in (1, 2, 4) if 6 * n * self.L <= sms] or [1])
            self.cl64 = self.ext.mnist_cl64_max_clusters(split) >= 1
            if self.cl64:
                self.S = split
        # CTAs per batch split: the cluster size of the cluster kernels, one CTA for the batch-split kernels
        self.ctas_per_split = 6 if self.tc else self.ext.mnist_cl64_cluster_ctas() if self.cl64 else 1
        self.kernel_name = (f"mnist_cl64_train_kernel<{64 // self.S}> (fp64 DMMA tiles, {self.S} x {self.ctas_per_split}-CTA cluster per node, DSMEM reduce)" if self.cl64 else
                            f"mnist_tc_train_kernel<{64 // self.S}> (3xTF32 mma.sync tiles, TMA tensor map, {self.S} x 6-CTA cluster per node)" if self.tc
                            else "convnet_generic_kernel (CUDA cores)" if self.generic else "mnist_kernel (mma.sync 3xTF32)")
        sh = problem.shards
        self.x = sh.x.reshape(sh.x.shape[0], -1).contiguous()
        assert self.x.shape[1] == 784
        self.x_is_u8 = self.x.dtype == torch.uint8
        if not self.x_is_u8:
            self.x = self.x.to(torch.float32).contiguous()
        self.y = sh.y.to(torch.int64).contiguous()
        mean, std = sh.norm if sh.norm is not None else (0.0, 1.0)
        self.shard_off = torch.tensor(sh.offsets[:-1], dtype=torch.int32, device=dev)
        self.shard_len = torch.tensor(sh.sizes, dtype=torch.int32, device=dev)
        self.calls = torch.zeros(self.L, dtype=torch.int32, device=dev)
        self.arrive = torch.zeros(self.L, dtype=torch.int32, device=dev)
        self.owns_calls = True      # the training kernel advances the draw counters (not the consensus kernels)
        self.grad_part = torch.zeros(self.L, self.S, self.n_pad, dtype=self.dtype, device=dev)
        self.loss_part = torch.zeros(self.L, self.S, dtype=torch.float32, device=dev)
        off = {s.name: s.offset for s in a.layout.slots}
        names = [s.name for s in a.layout.slots]
        self.base = dict(
            theta=a.theta.data_ptr(), n_pad=a.n_pad, L=self.L,
            off_wc=off[names[0]], off_bc=off[names[1]], off_w1=off[names[2]],
            off_b1=off[names[3]], off_w2=off[names[4]], off_b2=off[names[5]],
            x=self.x.data_ptr(), y=self.y.data_ptr(), x_is_u8=int(self.x_is_u8),
            mean=float(mean), inv_std=1.0 / float(std),
            direct=0, batch=self.B, seed=problem.seed, node0=pl.lo,
            shard_off=self.shard_off.data_ptr(), shard_len=self.shard_len.data_ptr(),
            calls=self.calls.data_ptr(), arrive=self.arrive.data_ptr(),
            grad_part=self.grad_part.data_ptr(), loss_part=self.loss_part.data_ptr(),
            spb=self.spb, S=self.S, tune=int(os.environ.get("NNDT_MNIST_TUNE", "1")),
            generic=int(self.generic), num_filters=spec.num_filters, kernel_size=spec.kernel_size,
            linear_width=spec.linear_width, dtype64=int(self.dtype == torch.float64), cl64=int(self.cl64))
        if self.tc:
            self.base.update(tc=1, w1_map=self.ext.make_w1_tensor_map(a.theta.data_ptr(), a.n_pad, self.L, off[names[2]]))
        if os.environ.get("NNDT_STEP_PROF") == "1":     # scripts/profile_round_phases.py
            self.step_prof = torch.zeros(self.L * self.S * self.ctas_per_split, 64, dtype=torch.int64, device=dev)
            self.base["step_prof"] = self.step_prof.data_ptr()
        self.train_op = self.ext.MnistOp(self.base)
        self._setup_eval()
        self.host_feed = None
        self.prev_op = None
        self._prev = None
        self._points = []       # every extra-point op (_point_op), in build order
        self.cross = []

    # ---- more points on the same minibatch (GT-HSGD, cross-gradient) --------
    def _point_op(self, theta_pt: torch.Tensor, grad_part: torch.Tensor) -> dict:
        """The training kernel on another parameter buffer ``theta_pt`` (``[L, n_pad]``, kept at this address) with its
        own partials ``grad_part``.  It draws the same minibatch as the training op because its draw counters
        (``calls``, ``arrive``) are a twin that the kernel advances in lockstep and ``sync_calls_from_host`` sets from
        the same host mirror; the fp32 cluster kernel gets its own W1 tensor map.  It stores no loss into the host
        mirror."""
        assert theta_pt.shape == self.pr.arena.theta.shape and theta_pt.dtype == self.dtype
        pt = dict(theta=theta_pt, calls=torch.zeros_like(self.calls), arrive=torch.zeros_like(self.arrive),
                  grad_part=grad_part, loss_part=torch.zeros_like(self.loss_part), direct=[])
        d = dict(self.base)
        d.pop("step_prof", None)
        d.update(theta=theta_pt.data_ptr(), calls=pt["calls"].data_ptr(), arrive=pt["arrive"].data_ptr(),
                 grad_part=grad_part.data_ptr(), loss_part=pt["loss_part"].data_ptr())
        if self.tc:
            a = self.pr.arena
            off_w1 = self.base["off_w1"]
            d.update(w1_map=self.ext.make_w1_tensor_map(theta_pt.data_ptr(), a.n_pad, self.L, off_w1))
        pt.update(base=d, op=self.ext.MnistOp(d))
        self._points.append(pt)
        self.sync_calls_from_host()
        if self.host_feed is not None:
            self._build_direct_point_ops(pt)
        return pt

    def _build_direct_point_ops(self, pt: dict):
        # the point's twins of the direct ops of step 0: the same stage slot, so the same staged minibatch
        pt["direct"] = []
        for b in range(2):
            d = dict(pt["base"])
            d.update(direct=1, x=self.x_stage[b, 0].data_ptr(), y=self.y_stage[b, 0].data_ptr(),
                     direct_bs=self.bs_stage[b, 0].data_ptr())
            pt["direct"].append(self.ext.MnistOp(d))

    def enable_prev_point(self, theta_prev: torch.Tensor):
        """Build the prev-point op (GT-HSGD) on ``theta_prev``: ``_point_op``."""
        pt = self._prev = self._point_op(theta_prev, torch.zeros_like(self.grad_part))
        self.theta_prev, self.prev_op = theta_prev, pt["op"]
        self.calls_prev, self.arrive_prev = pt["calls"], pt["arrive"]
        self.grad_part_prev, self.loss_part_prev = pt["grad_part"], pt["loss_part"]

    @property
    def direct_prev_ops(self):
        return self._prev["direct"] if self._prev is not None else []

    def enable_cross_points(self, theta_x: torch.Tensor):
        """Build one training op per slot of ``theta_x`` (``[P, L, n_pad]``, kept at this address), each a
        ``_point_op``; their partials are the slots of ``grad_part_x`` (``[P, L, S, n_pad]``)."""
        assert theta_x.dim() == 3 and theta_x.is_contiguous()
        self.theta_x = theta_x
        self.grad_part_x = torch.zeros((theta_x.shape[0],) + tuple(self.grad_part.shape), dtype=self.dtype,
                                       device=self.grad_part.device)
        self.cross = [self._point_op(theta_x[e], self.grad_part_x[e]) for e in range(theta_x.shape[0])]

    def launch_prev(self):
        """Enqueue the prev-point fwd+bwd on the batch the last ``launch`` drew (graph-capturable)."""
        self.prev_op.train()

    def launch_cross(self, e: int):
        """Enqueue the fwd+bwd at cross point ``e`` on the batch the last ``launch`` drew (graph-capturable)."""
        self.cross[e]["op"].train()

    def compute_grads_pair(self, theta_prev: torch.Tensor, grad_prev: torch.Tensor) -> torch.Tensor:
        """Eager API of ``ConsensusProblem.compute_grads_pair``: ``arena.grad`` at theta and ``grad_prev`` at the
        prev-point op's ``theta_prev``, on one draw."""
        assert self.prev_op is not None and theta_prev.data_ptr() == self.theta_prev.data_ptr()
        self.launch()
        self.launch_prev()
        torch.sum(self.grad_part_prev, dim=1, out=grad_prev)
        return self._collect_grads()

    def compute_grads_multi(self, points: torch.Tensor, grads: torch.Tensor) -> torch.Tensor:
        """Eager API of ``ConsensusProblem.compute_grads_multi`` on the cross-point ops' ``theta_x``."""
        assert self.cross and points.data_ptr() == self.theta_x.data_ptr()
        self.launch()
        for e in range(len(self.cross)):
            self.launch_cross(e)
        torch.sum(self.grad_part_x, dim=2, out=grads)
        return self._collect_grads()

    # ---- training ---------------------------------------------------------
    def launch(self):
        """Enqueue fwd+bwd of the next batch of every local node (graph-capturable).
        The draw counter is advanced by the consensus kernel that consumes the partials."""
        self.train_op.train()

    def compute_grads(self) -> torch.Tensor:
        """Eager API: fills ``arena.grad`` and advances the counters itself."""
        self.launch()
        return self._collect_grads()

    def _collect_grads(self) -> torch.Tensor:
        pr = self.pr
        torch.sum(self.grad_part, dim=1, out=pr.arena.grad)
        pr.count_draws_all(1)
        pr.last_losses = self.loss_part.sum(1).to(self.dtype)
        return pr.last_losses

    def sync_calls_from_host(self):
        pl = self.pr.placement
        self.calls.copy_(torch.as_tensor(self.pr.calls[pl.lo: pl.lo + pl.L].astype(np.int32)))
        for pt in self._points:
            pt["calls"].copy_(self.calls)

    # ---- host-fed batches (end-to-end input pipeline) -----------------------
    def enable_host_feed(self, steps_per_round: int, source: str):
        """Switch to a staged input pipeline: a staging kernel on a side stream gathers the *next* round's rows into
        one of two compact device staging sets (in-kernel sampler) while the current round computes, and the training
        kernel reads the staged batch by direct indexing.

        ``source="host"`` (``input_pipeline: host``, what ``bench.py`` times end to end): the dataset stays in pinned
        host memory and the staging kernel pulls the rows over PCIe (device-initiated H2D, no CPU work per round); the
        training kernel stores each step's losses straight into the pinned ``loss_host`` buffer.  ``source="device"``
        (``input_pipeline: staged``): the rows come from the HBM-resident shards, so the training kernel never runs the
        sampler chain or a random HBM gather on its critical path."""
        assert source in ("host", "device"), source
        pr, dev = self.pr, self.pr.device
        P, L, B = int(steps_per_round), self.L, self.B
        xb = 1 if self.x_is_u8 else 4
        if source == "host":
            self.host_x = self.x.cpu().contiguous().pin_memory()
            self.host_y = self.y.cpu().contiguous().pin_memory()
        else:
            self.host_x, self.host_y = self.x, self.y
        self.x_stage = torch.zeros(2, P, L, B, 784, dtype=self.x.dtype, device=dev)
        self.y_stage = torch.zeros(2, P, L, B, dtype=torch.int64, device=dev)
        self.bs_stage = torch.zeros(2, P, L, dtype=torch.int32, device=dev)
        self.loss_host = torch.zeros(L, self.S, dtype=torch.float32, pin_memory=True)
        # the training kernel stores each step's losses straight into this pinned host buffer over PCIe (no copy node on
        # the round's critical path); nothing crosses PCIe in the staged-resident pipeline
        self.loss_mode = "mirror" if source == "host" else "none"
        pl = pr.placement
        self.calls0 = torch.as_tensor(pr.calls[pl.lo: pl.lo + pl.L].astype(np.int32), device=dev)
        self.stage_round = torch.zeros(1, dtype=torch.int32, device=dev)
        self.stage_done = torch.zeros(1, dtype=torch.int32, device=dev)
        # a training CTA fills an SM's register file: a staging block that lands on an SM evicts a training CTA into a
        # second wave, so the staging grid is sized to the SMs left over by all L x S x ctas_per_split training CTAs
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        ctas = self.L * self.S * self.ctas_per_split
        free = sms - ctas if ctas <= sms else 0      # multi-wave grids leave no SM idle
        gather_blocks = int(os.environ.get("NNDT_GATHER_BLOCKS", "0")) or max(8, min(24, free - 2))
        self.direct_ops, self.gather_ops = [], []
        for b in range(2):
            ops = []
            for p in range(P):
                d = dict(self.base)
                d.update(direct=1, x=self.x_stage[b, p].data_ptr(), y=self.y_stage[b, p].data_ptr(),
                         direct_bs=self.bs_stage[b, p].data_ptr())
                if self.loss_mode == "mirror":
                    d.update(loss_mirror=self.loss_host.data_ptr())
                ops.append(self.ext.MnistOp(d))
            self.direct_ops.append(ops)
            self.gather_ops.append(self.ext.GatherOp(dict(
                x_host=self.host_x.data_ptr(), y_host=self.host_y.data_ptr(), row_bytes=784 * xb,
                x_stage=self.x_stage[b].data_ptr(), y_stage=self.y_stage[b].data_ptr(),
                bs_stage=self.bs_stage[b].data_ptr(), P=P, L=L, batch=B, seed=pr.seed, node0=pl.lo,
                shard_off=self.shard_off.data_ptr(), shard_len=self.shard_len.data_ptr(),
                calls0=self.calls0.data_ptr(), stage_round=self.stage_round.data_ptr(),
                done_ctr=self.stage_done.data_ptr(), max_blocks=gather_blocks)))
        # bench.py reads loader, loss_mode, loss_host and host_feed's mode / h2d_bytes / d2h_bytes for its e2e record
        self.loader = None
        self.host_feed = dict(P=P, mode="gpu_pull", source=source,
                              h2d_bytes=P * L * B * (784 * xb + 8) if source == "host" else 0,
                              d2h_bytes=L * self.S * 4 if source == "host" else 0)
        for pt in self._points:
            self._build_direct_point_ops(pt)
        return self.host_feed

    # ---- validation ---------------------------------------------------------
    def _setup_eval(self):
        pr = self.pr
        if pr.val is None:
            self.eval_op = None
            return
        dev = pr.device
        vx = pr.val.x.reshape(len(pr.val), -1).contiguous()
        self.vx = vx if vx.dtype == torch.uint8 else vx.to(torch.float32).contiguous()
        self.vy = pr.val.y.to(torch.int64).contiguous()
        V = len(pr.val)
        self.val_loss = torch.zeros(self.L, V, dtype=self.dtype, device=dev)
        self.val_correct = torch.zeros(self.L, V, dtype=torch.uint8, device=dev)
        mean, std = pr.val.norm if pr.val.norm is not None else (0.0, 1.0)
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        ctas = max(1, min(-(-V // SPB), sms // max(1, self.L)))
        d = dict(self.base)
        d.update(x=self.vx.data_ptr(), y=self.vy.data_ptr(), x_is_u8=int(self.vx.dtype == torch.uint8),
                 mean=float(mean), inv_std=1.0 / float(std), n_val=V,
                 val_loss=self.val_loss.data_ptr(), val_correct=self.val_correct.data_ptr(),
                 eval_ctas=ctas)
        self.eval_op = self.ext.MnistOp(d)

    def validate(self):
        self.eval_op.eval()
        return self.val_loss, self.val_correct.bool()
