"""The online sliding-window stream as the density training kernels draw it (ops/csrc/sampler.cuh, ``stream_row``),
transcribed to Python over the window table of ``data.sampler.window_table``, and the stream geometries and draw
counters that reach each of its branches.

``OnlineWindowSchedule.indices`` is the definition: it walks the unrolled window sequence from the stream position
``epoch * m + start`` of a batch.  The kernels instead fold the position into one period of the sequence (``q``
periods of ``P`` draws, offset ``r``), find the window by a linear search of the period's start offsets and key its
permutation by the global window index ``q * K + w`` (mod 2^32)."""
from __future__ import annotations

import numpy as np
import torch

from nn_distributed_training_b200.data.sampler import BatchSchedule, WIN_MAX, feistel_permute, mix_key

_M32 = 0xFFFFFFFF


def stream_rows(tab_row: np.ndarray, m: int, batch: int, call: int, seed: int, node: int, K: int = WIN_MAX):
    """Rows of a node's shard (offsets into it) the kernels draw at its ``call``-th batch: ``stream_row`` at every
    position of the batch, from the node's window table row."""
    epoch, start, size = BatchSchedule(m, batch).locate(call)
    n_win, period = int(tab_row[0]), int(tab_row[1])
    cum = tab_row[2: 2 + K + 1].astype(np.int64)
    lb = tab_row[2 + K + 1: 2 + 2 * K + 1].astype(np.int64)
    ub = tab_row[2 + 2 * K + 1: 2 + 3 * K + 1].astype(np.int64)
    d = epoch * m + start + np.arange(size, dtype=np.int64)          # first_draw + tt
    q, r = d // period, d % period
    # while (w + 1 < K && cum[w + 1] <= r) ++w;
    w = np.zeros(size, dtype=np.int64)
    for j in range(1, n_win):
        w += cum[j] <= r
    out = np.empty(size, dtype=np.int64)
    for qq, ww in sorted(set(zip(q.tolist(), w.tolist()))):
        sel = (q == qq) & (w == ww)
        key = mix_key(seed, node, (qq * n_win + ww) & _M32)
        pos = torch.as_tensor(r[sel] - cum[ww])
        out[sel] = lb[ww] + feistel_permute(pos, int(ub[ww] - lb[ww]), key).numpy()
    return out


def schedule_rows(schedule, m: int, batch: int, call: int, seed: int, node: int):
    """The same draw from the definition: what ``DistOnlineDensityProblem._draw_indices`` draws."""
    epoch, start, size = BatchSchedule(m, batch).locate(call)
    return schedule.indices(epoch * m + start, size, seed, node).numpy()


# (per-node (T scans, S points per scan, Wn scans per window), batch, per-launch draw counters of every node)
# Window geometry:  (20, 50, 3): K = 7 windows of 150 rows, P = m = 1000;  (10, 7, 3): K = 3, scan 9 is never drawn,
# P = 63 != m = 70;  (129, 3, 2): K = 64 = kWinMax, P = 384 != m = 387;  (2430, 500, 800): the paper's trajectory,
# K = 4, the last window 15 000 rows;  (2370, 500, 800): K = 3.
CASES = {
    # 0..99 inside window 0; 100..199 across the boundary at 150; epoch 1 (q = 1) at call 10
    "one_window_and_straddle": ([(20, 50, 3)], 100, [[0], [1], [10], [13]]),
    # B = 400 > 150 rows a window: each batch spans three or four windows; call 2 is the partial last batch of
    # epoch 0, call 3 the first of epoch 1
    "several_windows": ([(20, 50, 3)], 400, [[0], [1], [2], [3], [5]]),
    # the period wraps inside a batch: call 3 draws 60..69 across P = 63; calls 4 and 7 are epoch 1 (q = 1, 2)
    "period_wrap": ([(10, 7, 3)], 20, [[3], [4], [7], [11]]),
    # K = 64 windows of 6 rows: call 7 (350..386) crosses P = 384, later calls reach q = 1, 2
    "k64": ([(129, 3, 2)], 50, [[0], [7], [8], [15], [16]]),
    # nodes with different T and K in one launch, each at its own counter
    "mixed_nodes": ([(20, 50, 3), (10, 7, 3), (129, 3, 2)], 60, [[0, 0, 0], [2, 1, 6], [16, 3, 7], [17, 5, 13]]),
    # the paper's geometry: last (partial) batches, first batches of epoch 1, and stream positions past 2^32
    "paper_b12500": ([(2430, 500, 800), (2370, 500, 800)], 12500,
                     [[0, 31], [96, 94], [97, 95], [3600 * 98 + 97, 3700 * 95 + 31]]),
    "paper_b20000": ([(2430, 500, 800), (2370, 500, 800)], 20000,
                     [[60, 59], [61, 60], [19, 20], [3600 * 61 + 60, 3700 * 60 + 59]]),
}
