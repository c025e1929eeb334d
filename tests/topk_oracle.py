"""NumPy oracle of the top-k code rows of CHOCO-SGD and BEER (``compressor: topk``), written from the layout and the
selection rule of ``csrc/consensus.h``; it does not call ``ops/consensus_ref.py``."""
from __future__ import annotations

import numpy as np


def topk_select(v: np.ndarray, live: np.ndarray, k: int) -> np.ndarray:
    """Indices (ascending) of the k live elements of one row with the largest |v|, ties to the smaller index: keys are
    the IEEE bits with the sign bit cleared, ordered with np.lexsort on (index, -key)."""
    v = np.ascontiguousarray(v)
    bits = v.view(np.uint64 if v.dtype == np.float64 else np.uint32).astype(np.uint64)
    key = (bits & np.uint64(0x7FFFFFFFFFFFFFFF if v.dtype == np.float64 else 0x7FFFFFFF)).astype(np.int64)
    cand = np.nonzero(live)[0]
    order = cand[np.lexsort((cand, -key[cand]))]
    return np.sort(order[:k])


def topk_decode(row: np.ndarray, n_pad: int, dtype, k: int):
    """dec(q) of one top-k code row (uint8) as float64, its indices and values: k values of ``dtype``, then k uint32
    indices, then zero padding."""
    dt = np.dtype(dtype)
    row = np.ascontiguousarray(row)
    vals = row[: k * dt.itemsize].view(dt)
    idx = row[k * dt.itemsize: k * (dt.itemsize + 4)].view("<u4")
    d = np.zeros(n_pad)
    d[idx] = vals.astype(np.float64)
    return d, idx, vals
