"""Stateless, device-side batch sampling.

The reference draws minibatches through a Python ``DataLoader`` per node
(problems/dist_mnist_problem.py:45-54,83-88): shuffle each epoch, last batch
partial, re-arm on ``StopIteration``.  In this framework a batch is a pure
function of ``(seed, node, call index)``:

* ``BatchSchedule`` gives, for the c-th draw of a node, the epoch, the start
  position inside the epoch's permutation and the batch size (same epoch /
  partial-batch structure as the DataLoader),
* the epoch permutation is a keyed 4-round Feistel network with cycle walking
  (``feistel_permute``): no stored index list, no host work per step, and the
  sm_90a kernels evaluate the identical function in registers
  (ops/csrc/sampler.cuh) so the whole training round can live in a CUDA graph.

``OnlineWindowSchedule`` re-expresses the sliding-window logic of
``OnlineTrajectoryLidarDataset`` (floorplans/lidar/lidar.py:397-424) as index
arithmetic over the draw counter.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import torch

_M32 = 0xFFFFFFFF
_C1 = 0x9E3779B1
_C2 = 0x85EBCA6B
_ROUND_KEYS = (0xA511E9B3, 0x63D83595, 0x1B873593, 0xCC9E2D51)


def mix_key(seed: int, node: int, epoch: int) -> int:
    """32-bit key for (seed, node, epoch) — identical in sampler.cuh."""
    x = (seed * 0x9E3779B1 + node * 0x85EBCA77 + epoch * 0xC2B2AE3D + 0x27D4EB2F) & _M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & _M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & _M32
    x ^= x >> 16
    return x


def _half_bits(m: int) -> int:
    bits = max(2, int(m - 1).bit_length())
    return (bits + 1) // 2


def _round_fn(x: torch.Tensor, k: int, mask: int) -> torch.Tensor:
    x = ((x ^ k) * _C1) & _M32
    x = x ^ (x >> 15)
    x = (x * _C2) & _M32
    x = x ^ (x >> 13)
    return x & mask


def feistel_permute(pos: torch.Tensor, m: int, key: int) -> torch.Tensor:
    """Bijection of ``[0, m)`` applied elementwise to int64 ``pos`` (values < m)."""
    if m <= 1:
        return torch.zeros_like(pos)
    h = _half_bits(m)
    mask = (1 << h) - 1
    x = pos.clone().to(torch.int64)
    todo = torch.ones_like(x, dtype=torch.bool)
    while bool(todo.any()):
        cur = x[todo]
        left, right = cur >> h, cur & mask
        for r in range(4):
            left, right = right, left ^ _round_fn(right, (key + _ROUND_KEYS[r]) & _M32, mask)
        cur = (left << h) | right
        x[todo] = cur
        todo = todo.clone()
        todo[todo.clone()] = cur >= m
    return x


@dataclass
class BatchSchedule:
    """DataLoader-equivalent batching of a dataset of ``m`` samples."""

    m: int
    batch_size: int

    @property
    def batches_per_epoch(self) -> int:
        return max(1, -(-self.m // self.batch_size))

    def locate(self, call: int) -> Tuple[int, int, int]:
        """(epoch, start, size) of the ``call``-th draw (0-based)."""
        bpe = self.batches_per_epoch
        epoch, b = divmod(call, bpe)
        start = b * self.batch_size
        return epoch, start, min(self.batch_size, self.m - start)

    def epochs_completed(self, calls: int) -> int:
        """Value of the reference's ``epoch_tracker`` after ``calls`` draws: it
        is bumped when a draw hits ``StopIteration`` (dist_mnist_problem.py:85-88)."""
        return 0 if calls <= 0 else (calls - 1) // self.batches_per_epoch

    def indices(self, call: int, seed: int, node: int, device="cpu") -> torch.Tensor:
        epoch, start, size = self.locate(call)
        pos = torch.arange(start, start + size, dtype=torch.int64, device=device)
        return feistel_permute(pos, self.m, mix_key(seed, node, epoch))


class OnlineWindowSchedule:
    """Sliding-window stream over ``num_scans`` scans of ``scan_size`` points.

    Window w covers points ``[lb_w, ub_w)``; draws consume a keyed permutation
    of the window and move on when it is exhausted.  ``scan_cursor`` after a
    window switch indexes the robot position (``curr_pos``) exactly as in the
    reference (lidar.py:403-422).
    """

    def __init__(self, num_scans: int, scan_size: int, scans_in_window: int):
        self.T, self.S, self.Wn = int(num_scans), int(scan_size), int(scans_in_window)
        # the window sequence is periodic; unroll one period lazily
        self._windows: List[Tuple[int, int, int]] = []  # (lb, ub, scan_cursor_after)
        self._cursor = 0
        self._cum = [0]

    def _extend(self):
        cur, T, Wn, S = self._cursor, self.T, self.Wn, self.S
        if cur + Wn >= T:
            if cur == T - 1:
                cur = Wn
                lb, ub = S * (cur - Wn), S * cur
            else:
                lb, ub = S * cur, S * T
                cur = T - 1
        else:
            cur += Wn
            lb, ub = S * (cur - Wn), S * cur
        self._cursor = cur
        self._windows.append((lb, ub, cur))
        self._cum.append(self._cum[-1] + (ub - lb))

    def window(self, w: int) -> Tuple[int, int, int]:
        while len(self._windows) <= w:
            self._extend()
        return self._windows[w]

    def locate_draw(self, draw: int) -> Tuple[int, int]:
        """(window index, offset inside window) of the ``draw``-th sample."""
        while self._cum[-1] <= draw:
            self._extend()
        w = int(np.searchsorted(np.asarray(self._cum), draw, side="right")) - 1
        return w, draw - self._cum[w]

    def scan_cursor_at(self, draws_done: int) -> int:
        """Scan index whose pose is ``curr_pos`` after ``draws_done`` samples were
        drawn.  The reference switches window lazily (on the first draw that
        finds the list empty), so after exactly exhausting window w the pose
        is still window w's."""
        if draws_done <= 0:
            return self.window(0)[2]
        w, _ = self.locate_draw(draws_done - 1)
        return self.window(w)[2]

    def indices(self, first_draw: int, count: int, seed: int, node: int, device="cpu") -> torch.Tensor:
        out = []
        d, left = first_draw, count
        while left > 0:
            w, off = self.locate_draw(d)
            lb, ub, _ = self.window(w)
            take = min(left, (ub - lb) - off)
            pos = torch.arange(off, off + take, dtype=torch.int64, device=device)
            out.append(lb + feistel_permute(pos, ub - lb, mix_key(seed, node, w)))
            d += take
            left -= take
        return torch.cat(out)


WIN_MAX = 64   # windows per period the in-kernel sampler holds (kWinMax in ops/csrc/sampler.cuh)


def window_table(schedules: List[OnlineWindowSchedule], K: int = WIN_MAX) -> np.ndarray:
    """Per-node tables of one period of each sliding-window stream, the layout ``stream_row`` of
    ops/csrc/sampler.cuh decodes: row ``l`` is ``[n_windows, period, cum[0..K], lb[K], ub[K]]`` for
    ``schedules[l]``, where ``cum`` are the window start offsets in the period.  The period ends at
    the first recurrence of window 0."""
    tab = np.zeros((len(schedules), 2 + (K + 1) + 2 * K), dtype=np.int64)
    for l, sch in enumerate(schedules):
        wins = [sch.window(0)]
        while True:
            w = sch.window(len(wins))
            if w == wins[0]:
                break
            wins.append(w)
            if len(wins) > K:
                raise RuntimeError(f"online window stream has more than {K} windows per period")
        cum = np.concatenate([[0], np.cumsum([ub - lb for lb, ub, _ in wins])])
        tab[l, 0], tab[l, 1] = len(wins), cum[-1]
        tab[l, 2: 2 + len(cum)] = cum
        tab[l, 2 + K + 1: 2 + K + 1 + len(wins)] = [w[0] for w in wins]
        tab[l, 2 + 2 * K + 1: 2 + 2 * K + 1 + len(wins)] = [w[1] for w in wins]
    return tab
