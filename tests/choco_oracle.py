"""Float64 oracle of CHOCO-SGD's gossip and step (``choco_mix`` / ``choco_step`` of ``ops/csrc/consensus.cu``), written
in NumPy from the algorithm and the code-row layout of ``csrc/consensus.h``; it does not call ``ops/consensus_ref.py``.

Arrays are ``[N, n_pad]`` float64; code rows are ``uint8 [code_bytes]``.  Each step returns its result and a first-order
error bound ``err`` in the style of ``consensus_oracle.py`` (every rounding charged one unit ``u`` of the kernel's dtype).
"""
from __future__ import annotations

import numpy as np

BLOCK = 32


def decode(row: np.ndarray, compressor: str, n_pad: int, dtype, live: np.ndarray):
    """dec(q) of one code row (uint8) as float64, and its rounding bound in units of |dec| (int8: code * scale is
    rounded once in ``dtype``; the other formats decode exactly)."""
    dt = np.dtype(dtype)
    nb = n_pad // BLOCK
    row = np.ascontiguousarray(row)
    if compressor == "none":
        return row[: n_pad * dt.itemsize].view(dt).astype(np.float64), 0.0
    if compressor == "int8":
        q = row[:n_pad].view(np.int8).astype(np.float64)
        sc = row[n_pad: n_pad + nb * dt.itemsize].view(dt).astype(np.float64)
        return q * np.repeat(sc, BLOCK), 1.0
    words = row[: 4 * nb].view("<u4")
    sc = row[4 * nb: 4 * nb + nb * dt.itemsize].view(dt).astype(np.float64)
    e = np.arange(n_pad)
    bit = (words[e // BLOCK] >> (e % BLOCK).astype(np.uint32)) & 1
    return np.where(live, np.where(bit == 1, 1.0, -1.0) * np.repeat(sc, BLOCK), 0.0), 0.0


def mix(theta, x_hat, s, dec, nbrs, W, gamma, u, rel_dec):
    """s_i += W_ii dec_i + sum_j W_ij dec_j; theta_i += gamma (s_i - x_hat_i)."""
    N = theta.shape[0]
    th, sn = theta.copy(), s.copy()
    e_th, e_s = np.zeros_like(theta), np.zeros_like(s)
    for i in range(N):
        t = W[i, i] * dec[i]
        mag = np.abs(t)
        for j in nbrs[i]:
            t = t + W[i, j] * dec[j]
            mag += np.abs(W[i, j] * dec[j])
        e_t = u * (mag * (1.0 + rel_dec) + np.abs(t))
        sn[i] = s[i] + t
        e_s[i] = e_t + u * np.abs(sn[i])
        d = sn[i] - x_hat[i]
        th[i] = theta[i] + gamma * d
        e_th[i] = gamma * (e_s[i] + u * np.abs(d)) + u * (gamma * np.abs(d) + np.abs(th[i]))
    return th, sn, e_th, e_s


def sign_scale(v: np.ndarray, live: np.ndarray, u: float):
    """sum |v| / n_live per block over the live elements (0 for a block without one), and the round-off bound of a
    32-term sum and one division."""
    a = np.where(live, np.abs(v), 0.0).reshape(v.shape[:-1] + (-1, BLOCK))
    nl = live.reshape(-1, BLOCK).sum(-1)
    tot = a.sum(-1)
    sc = np.where(nl > 0, tot / np.maximum(nl, 1), 0.0)
    return sc, u * (BLOCK + 1) * sc


def contraction_delta(v: np.ndarray, compressor: str, live: np.ndarray) -> float:
    """The delta of the compressor's contraction ||dec(Q(v)) - v||^2 <= (1 - delta) ||v||^2 on one block."""
    if compressor == "none":
        return 1.0
    if compressor == "int8":
        return 1.0 - BLOCK / 254.0 ** 2
    n = max(int(live.sum()), 1)
    l1, l2 = np.abs(v[live]).sum(), (v[live] ** 2).sum()
    return l1 * l1 / (n * l2) if l2 > 0 else 1.0
