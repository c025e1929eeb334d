"""Float64 oracle of generalized advantage estimation, GAE(lambda), and its round-off bound.

Rows ``r = (blk * T + c) * E + e``; per (block, world) scan backwards over the block's ``T`` cycles:

    delta_c = r_c + gamma V_{c+1} - V_c,   A_c = delta_c + gamma lam A_{c+1},   G_c = A_c + V_c,   V_T = A_T = 0.

``gae64`` evaluates that in float64 with numpy; ``gae_same_order`` evaluates it in a given numpy dtype with one
rounding per operation in the order written (what the sm_90a scan and the torch path do), so a batch-dtype result
can be held to it bit for bit.

Round-off bound: a step rounds five results (gamma V, the two sums of delta, gamma lam A, their sum) plus the
inputs gamma and gamma lam, each within ``u |result|``, and every result of step c is at most
``S_c = (|r_c| + gamma |V_{c+1}| + |V_c|) + gamma lam S_{c+1}``.  So the local error of step c is at most ``6 u S_c``
to first order, and it reaches step c' < c damped by (gamma lam)^(c - c'):

    |A_c - A64_c| <= B_c,   B_c = 8 u S_c + gamma lam B_{c+1}                  (8 = 6, doubled for the 2nd order)
    |G_c - G64_c| <= B_c + 2 u (|A_c| + |V_c|).
"""
from __future__ import annotations

import numpy as np

U = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}


def _blocks(x, T, E):
    x = np.asarray(x)
    if x.shape[-1] % (T * E):
        raise ValueError(f"T * E = {T} * {E} does not divide R = {x.shape[-1]}")
    return x.reshape(-1, T, E)


def gae64(rews, values, gamma, lam, T, E):
    """``(A, G)`` in float64, shaped like ``rews``."""
    shape = np.shape(rews)
    r = _blocks(rews, T, E).astype(np.float64)
    v = _blocks(values, T, E).astype(np.float64)
    A = np.zeros_like(r)
    nxt_a = np.zeros_like(r[:, 0])
    nxt_v = np.zeros_like(r[:, 0])
    for c in range(T - 1, -1, -1):
        nxt_a = r[:, c] + gamma * nxt_v - v[:, c] + gamma * lam * nxt_a
        A[:, c] = nxt_a
        nxt_v = v[:, c]
    return A.reshape(shape), (A + v).reshape(shape)


def gae_same_order(rews, values, gamma, lam, T, E, dtype):
    """``(A, G)`` in ``dtype`` (np.float32 / np.float64) with one rounding per operation:
    ``A_c = ((r_c + g * V_{c+1}) - V_c) + gl * A_{c+1}`` with ``g = dtype(gamma)``, ``gl = dtype(gamma * lam)``."""
    shape = np.shape(rews)
    r = _blocks(rews, T, E).astype(dtype)
    v = _blocks(values, T, E).astype(dtype)
    g, gl = dtype(gamma), dtype(gamma * lam)
    A = np.zeros_like(r)
    a = np.zeros_like(r[:, 0])
    vn = np.zeros_like(r[:, 0])
    for c in range(T - 1, -1, -1):
        delta = (r[:, c] + g * vn) - v[:, c]
        a = delta + gl * a
        A[:, c] = a
        vn = v[:, c]
    return A.reshape(shape), (A + v).reshape(shape)


def bound(rews, values, gamma, lam, T, E, u):
    """``(B_A, B_G)``: elementwise round-off bounds of a computation with unit round-off ``u`` from the same inputs."""
    shape = np.shape(rews)
    r = np.abs(_blocks(rews, T, E).astype(np.float64))
    v = np.abs(_blocks(values, T, E).astype(np.float64))
    gl = gamma * lam
    S = np.zeros_like(r)
    B = np.zeros_like(r)
    s = np.zeros_like(r[:, 0])
    b = np.zeros_like(r[:, 0])
    vn = np.zeros_like(r[:, 0])
    for c in range(T - 1, -1, -1):
        s = (r[:, c] + gamma * vn + v[:, c]) + gl * s
        b = 8 * u * s + gl * b
        S[:, c], B[:, c] = s, b
        vn = v[:, c]
    BG = B + 2 * u * (S + v)
    return B.reshape(shape), BG.reshape(shape)


def rtgs64(rews, gamma, T, E):
    """Float64 rewards-to-go of every (block, world)."""
    shape = np.shape(rews)
    r = _blocks(rews, T, E).astype(np.float64)
    out = np.zeros_like(r)
    run = np.zeros_like(r[:, 0])
    for c in range(T - 1, -1, -1):
        run = r[:, c] + gamma * run
        out[:, c] = run
    return out.reshape(shape)


def normalise64(A):
    """Per row of ``A [N, R]``: ``(A - mean) / (std + 1e-10)`` with the unbiased std, in float64."""
    A = np.asarray(A, dtype=np.float64)
    return (A - A.mean(-1, keepdims=True)) / (A.std(-1, ddof=1, keepdims=True) + 1e-10)


def normalised_bound(A64, BA, u):
    """Bound on ``|adv - normalise64(A64)|`` (max over a row) for a normalisation in unit round-off ``u`` of an ``A``
    within ``BA`` of ``A64``: the shift of the mean and of the std by the input error, over the std, plus the
    normalisation's own rounding."""
    A64 = np.asarray(A64, dtype=np.float64)
    sd = A64.std(-1, ddof=1, keepdims=True)
    z = np.abs(A64 - A64.mean(-1, keepdims=True)) / sd
    return (2 * BA.max(-1, keepdims=True) * (1 + z)) / sd + 16 * u * (1 + z)
