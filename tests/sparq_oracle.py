"""Float64 oracle of SPARQ-SGD's three launches (``sparq_mix`` / ``sparq_step`` / ``sparq_publish`` of
``ops/csrc/consensus.cu``), written in NumPy from the algorithm and the row layout of ``csrc/consensus.h``; it does not
call ``ops/consensus_ref.py``.  Code bodies are decoded with ``choco_oracle.decode`` (the layout is CHOCO's).

Arrays are ``[N, n_pad]`` float64; rows are ``uint8 [row_bytes]``.  Each launch returns its result and a first-order
error bound ``err`` in the style of ``consensus_oracle.py`` (every rounding charged one unit ``u`` of the kernel's
dtype; the float64 sums of the trigger test one unit ``U64`` each).
"""
from __future__ import annotations

import numpy as np

import choco_oracle as cho

TAIL = 16
U64 = 2.0 ** -53


def row_bytes(code_bytes: int) -> int:
    """The code row and the 16-byte tail, rounded up to 16."""
    return -(-(code_bytes + TAIL) // 16) * 16


def tail(row: np.ndarray, code_bytes: int):
    """(trig, reserved word, e) of one row's tail."""
    t = np.ascontiguousarray(row[code_bytes: code_bytes + TAIL])
    w = t[:8].view("<u4")
    return int(w[0]), int(w[1]), float(t[8:].view("<f8")[0])


def threshold(c0: float, growth: float, alphas) -> np.ndarray:
    """thr_k = c0 (k + 1)^growth alpha_k^2."""
    return np.array([c0 * (k + 1) ** growth * a * a for k, a in enumerate(alphas)], dtype=np.float64)


def mix(theta, x_hat, s, dec, trig, nbrs, W, gamma, u, rel_dec):
    """s_i += sum over j in {i} u N_i with trig_j of W_ij dec_j (own term first); theta_i += gamma (s_i - x_hat_i)."""
    N = theta.shape[0]
    th, sn = theta.copy(), s.copy()
    e_th, e_s = np.zeros_like(theta), np.zeros_like(s)
    for i in range(N):
        t = np.zeros(theta.shape[1])
        mag = np.zeros(theta.shape[1])
        for j in [i] + list(nbrs[i]):
            if trig[j]:
                t = t + W[i, j] * dec[j]
                mag += np.abs(W[i, j] * dec[j])
        e_t = u * (mag * (1.0 + rel_dec) + np.abs(t))
        sn[i] = s[i] + t
        e_s[i] = e_t + u * np.abs(sn[i])
        d = sn[i] - x_hat[i]
        th[i] = theta[i] + gamma * d
        e_th[i] = gamma * (e_s[i] + u * np.abs(d)) + u * (gamma * np.abs(d) + np.abs(th[i]))
    return th, sn, e_th, e_s


def step(theta, g, e_g, alpha, u):
    """theta -= alpha g, one fused multiply-add per element."""
    th = theta - alpha * g
    return th, alpha * e_g + u * (np.abs(theta) + 2.0 * alpha * np.abs(g))


def sqdist(theta, x_hat, u):
    """e_i = sum (theta_i - x_hat_i)^2 with the difference rounded in the kernel's dtype (unit u) and the squares and
    the sum in float64: relative bound 2 u + n_pad U64."""
    d = theta - x_hat
    e = (d * d).sum(1)
    return e, (2.0 * u + (theta.shape[1] + 2) * U64) * e


def publish(e, thr):
    """trig_i = e_i > thr."""
    return e > thr
