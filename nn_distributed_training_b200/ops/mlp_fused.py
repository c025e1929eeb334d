"""Python side of the tensor-core MLP kernels: csrc/mlp_tc.cu (float32 arm: bf16 operands, fp32 accumulation) and
csrc/mlp_f64.cu (float64 arm: fp64 DMMA tiles on 2-CTA clusters)."""
from __future__ import annotations

import numpy as np
import torch

from . import load_ext
from ..data.sampler import WIN_MAX, window_table
from ..models.spec import MLPSpec

FIRST = {"relu": 0, "sin_relu": 1}
LAST = {"none": 0, "sigmoid": 1}
LOSS = {"BCELoss": 0, "MSELoss": 1, "L1Loss": 2}
TRAIN_KERNEL_READY = True


def shape_supported(spec: MLPSpec) -> bool:
    s = spec.shape
    return (len(s) == 6 and s[0] == 2 and s[1] in (64, 128, 256) and tuple(s[2:5]) == (64, 64, 64) and s[5] == 1
            and spec.first in FIRST and spec.hidden == "relu" and spec.last in LAST)


def supports(spec: MLPSpec, base_loss, dtype=torch.float32) -> bool:
    return (TRAIN_KERNEL_READY and dtype in (torch.float32, torch.float64) and shape_supported(spec)
            and type(base_loss).__name__ in LOSS and getattr(base_loss, "reduction", "mean") == "mean")


F64_TILE = 32      # rows of a cluster tile of the float64 kernels


def f64_max_clusters(ext, h1: int) -> int:
    """Co-resident 2-CTA clusters of the float64 training kernel; an error if it cannot launch at all."""
    n = ext.mlp_f64_max_clusters(h1)
    if n < 1:
        raise RuntimeError(f"the float64 MLP kernel (h1={h1}) cannot be launched on this device")
    return n


def op_dict(arena, spec: MLPSpec, L: int):
    off = [s.offset for s in arena.layout.slots]
    assert len(off) == 10
    if arena.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"no fused MLP kernel for {arena.dtype}")
    return dict(theta=arena.theta.data_ptr(), n_pad=arena.n_pad, L=L, off=off, d_in=spec.shape[0], h1=spec.shape[1],
                first_act=FIRST[spec.first], last_act=LAST[spec.last], scale=float(spec.scale),
                dtype64=int(arena.dtype == torch.float64))


class MlpForward:
    """Forward-only evaluation of every local node's network on shared inputs ``x [M, d_in]``."""

    def __init__(self, arena, spec: MLPSpec, L: int, device):
        self.ext = load_ext(required=True)
        self.arena, self.spec, self.L, self.device = arena, spec, L, device
        self.dtype = arena.dtype
        self.sms = torch.cuda.get_device_properties(device).multi_processor_count
        if self.dtype == torch.float64:
            self.max_clusters = f64_max_clusters(self.ext, spec.shape[1])
        self._cache = {}

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        x = x.to(self.dtype).contiguous()
        M = x.shape[0]
        out = torch.empty(self.L, M, dtype=self.dtype, device=self.device)
        d = op_dict(self.arena, self.spec, self.L)
        if self.dtype == torch.float64:      # 2-CTA clusters per node: one wave over all nodes
            ctas = max(1, min(-(-M // F64_TILE), self.max_clusters // max(1, self.L)))
        else:
            ctas = max(1, min(-(-M // 128), max(1, (2 * self.sms) // max(1, self.L))))
        d.update(x=x.data_ptr(), n_rows=M, out=out.data_ptr(), fwd_ctas=ctas)
        op = self.ext.MlpOp(d)
        op.forward()
        self._keep = (x, out, op)
        return out


class FusedMLP:
    """Fused training/eval engine of a density problem (FourierNet family) — the analogue of
    ``FusedMnist``: device-resident shards, stateless sampling, per-CTA gradient partials that
    the consensus update kernel sums."""

    def __init__(self, problem):
        self.pr = problem
        self.ext = load_ext(required=True)
        dev = problem.device
        a, pl = problem.arena, problem.placement
        self.spec = problem.base_model.spec
        self.L, self.n_pad, self.B = pl.L, a.n_pad, problem.train_batch_size
        self.dtype = a.dtype
        self.sms = torch.cuda.get_device_properties(dev).multi_processor_count
        if self.dtype == torch.float64:
            # G 2-CTA clusters over the L x ceil(B / 32) tiles; each CTA of a cluster owns one partial row
            tmax = -(-self.B // F64_TILE)
            self.G = max(1, min(f64_max_clusters(self.ext, self.spec.shape[1]), self.L * tmax))
            self.S = 2 * (-(-self.G // self.L) + 1)
        else:
            tmax = -(-self.B // 128)
            self.G = max(1, min(self.sms, self.L * tmax))
            self.S = -(-self.G // self.L) + 1
        sh = problem.shards
        self.x = sh.x.to(self.dtype).contiguous()
        self.y = sh.y.to(self.dtype).contiguous()
        self.shard_off = torch.tensor(sh.offsets[:-1], dtype=torch.int32, device=dev)
        self.shard_len = torch.tensor(sh.sizes, dtype=torch.int32, device=dev)
        self.calls = torch.zeros(self.L, dtype=torch.int32, device=dev)
        self.grad_part = torch.zeros(self.L, self.S, self.n_pad, dtype=self.dtype, device=dev)
        self.loss_part = torch.zeros(self.L, self.S, dtype=self.dtype, device=dev)
        self.win_table = self._window_table()
        d = op_dict(a, self.spec, self.L)
        d.update(win_table=None if self.win_table is None else self.win_table.data_ptr())
        d.update(loss=LOSS[type(problem.base_loss).__name__], x=self.x.data_ptr(), y=self.y.data_ptr(),
                 direct=0, batch=self.B, seed=problem.seed, node0=pl.lo,
                 shard_off=self.shard_off.data_ptr(), shard_len=self.shard_len.data_ptr(),
                 calls=self.calls.data_ptr(), grad_part=self.grad_part.data_ptr(),
                 loss_part=self.loss_part.data_ptr(), S=self.S, train_ctas=self.G)
        self.base = d
        self.train_op = self.ext.MlpOp(d)
        self._fwd = MlpForward(a, self.spec, self.L, dev)
        self.host_feed = None
        self.prev_op = None
        self.cross = []

    def _point_op(self, theta_pt: torch.Tensor, grad_part: torch.Tensor):
        """The training kernel on another parameter buffer ``theta_pt`` (``[L, n_pad]``, kept at this address) with its
        own partials ``grad_part``.  It reads the same draw counters ``calls`` as the training op, which the consensus
        step advances after every launch of the round, so it draws the same minibatch.  It leaves the loss EMA alone."""
        assert theta_pt.shape == self.pr.arena.theta.shape and theta_pt.dtype == self.dtype
        loss_part = torch.zeros_like(self.loss_part)
        d = dict(self.base)
        d.update(theta=theta_pt.data_ptr(), grad_part=grad_part.data_ptr(), loss_part=loss_part.data_ptr())
        return self.ext.MlpOp(d), loss_part

    def enable_prev_point(self, theta_prev: torch.Tensor):
        """Build the prev-point op (GT-HSGD) on ``theta_prev``: ``_point_op``."""
        self.theta_prev = theta_prev
        self.grad_part_prev = torch.zeros_like(self.grad_part)
        self.prev_op, self.loss_part_prev = self._point_op(theta_prev, self.grad_part_prev)

    def enable_cross_points(self, theta_x: torch.Tensor):
        """Build one training op per slot of ``theta_x`` (``[P, L, n_pad]``, kept at this address), each a
        ``_point_op``; their partials are the slots of ``grad_part_x`` (``[P, L, S, n_pad]``)."""
        assert theta_x.dim() == 3 and theta_x.is_contiguous()
        self.theta_x = theta_x
        self.grad_part_x = torch.zeros((theta_x.shape[0],) + tuple(self.grad_part.shape), dtype=self.dtype,
                                       device=self.grad_part.device)
        self.cross = [self._point_op(theta_x[e], self.grad_part_x[e]) for e in range(theta_x.shape[0])]

    WIN_MAX = WIN_MAX

    def _window_table(self):
        """Online problems: per-node tables of one period of the sliding-window stream
        (``data.sampler.OnlineWindowSchedule``) for the in-kernel sampler."""
        pr = self.pr
        dsets = getattr(pr, "_datasets", None)
        if dsets is None or not hasattr(dsets[0], "schedule"):
            return None
        tab = window_table([dsets[g].schedule for g in pr.placement.local_nodes], self.WIN_MAX)
        return torch.as_tensor(tab, device=pr.device)

    ema_in_kernel = False   # set by the consensus engine when its kernels maintain the loss EMA

    def launch(self):
        self.train_op.train()
        if getattr(self.pr, "track_tloss", False) and not self.ema_in_kernel:
            # device-side EMA of the training loss (capturable: no host sync)
            self.pr._ema_update(self.pr.tloss_local, self.loss_part.sum(1))

    def launch_prev(self):
        """Enqueue the prev-point fwd+bwd on the batch of the last ``launch`` (graph-capturable)."""
        self.prev_op.train()

    def compute_grads_pair(self, theta_prev: torch.Tensor, grad_prev: torch.Tensor) -> torch.Tensor:
        """Eager API of ``ConsensusProblem.compute_grads_pair``: both launches on one draw, then ``compute_grads``'s
        bookkeeping once."""
        assert self.prev_op is not None and theta_prev.data_ptr() == self.theta_prev.data_ptr()
        self.launch()
        self.launch_prev()
        torch.sum(self.grad_part_prev, dim=1, out=grad_prev)
        return self._collect_grads()

    def launch_cross(self, e: int):
        """Enqueue the fwd+bwd at cross point ``e`` on the batch of the last ``launch`` (graph-capturable)."""
        self.cross[e][0].train()

    def compute_grads_multi(self, points: torch.Tensor, grads: torch.Tensor) -> torch.Tensor:
        """Eager API of ``ConsensusProblem.compute_grads_multi`` on the cross-point ops' ``theta_x``."""
        assert self.cross and points.data_ptr() == self.theta_x.data_ptr()
        self.launch()
        for e in range(len(self.cross)):
            self.launch_cross(e)
        torch.sum(self.grad_part_x, dim=2, out=grads)
        return self._collect_grads()

    def compute_grads(self) -> torch.Tensor:
        self.launch()
        return self._collect_grads()

    def _collect_grads(self) -> torch.Tensor:
        pr = self.pr
        torch.sum(self.grad_part, dim=1, out=pr.arena.grad)
        self.calls += 1
        pr.count_draws_all(1)
        pr.last_losses = self.loss_part.sum(1)
        if getattr(pr, "track_tloss", False) and self.ema_in_kernel:
            pr._ema_update(pr.tloss_local, pr.last_losses)   # eager API: no consensus kernel follows
        return pr.last_losses

    def sync_calls_from_host(self):
        pl = self.pr.placement
        self.calls.copy_(torch.as_tensor(self.pr.calls[pl.lo: pl.lo + pl.L].astype(np.int32)))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self._fwd(x)
