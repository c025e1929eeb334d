"""Float64 NumPy oracle of Gossip-PGA (optimizers/gossip_pga.py), written from the equations, not from consensus_ref.

Round k of every node, with the mixing matrix W_k of the round and DSGD's step schedule alpha_k:

    global round (k mod period == period - 1):  theta <- 1 1^T theta / N
    gossip round:                               theta <- W_k theta  (gossip), theta  (local SGD)
    theta <- theta - alpha_k grad(theta, k)

One function per fused launch, each returning its result and a first-order error bound (in the style of
``tests/consensus_oracle.py``): ``pga_sum`` (a rank's float64 partial sum), ``pga_mix`` (either branch) and
``dsgd_step``."""
from __future__ import annotations

import numpy as np

U64 = 2.0 ** -53


def is_global(k: int, period: int) -> bool:
    return k % period == period - 1


def run(theta0: np.ndarray, Ws, alphas, period: int, gossip: bool, grad, rounds: int):
    """Yield ``theta`` after every round; ``grad(x, k)`` is the ``[N, n]`` gradient of every node at points ``x`` on
    draw k, ``Ws[k]`` the round's matrix and ``alphas[k]`` its step."""
    theta = np.array(theta0, dtype=np.float64)
    for k in range(rounds):
        if is_global(k, period):
            theta = np.repeat(theta.mean(0, keepdims=True), theta.shape[0], axis=0)
        elif gossip:
            theta = Ws[k] @ theta
        theta = theta - alphas[k] * grad(theta, k)
        yield theta.copy()


def pga_sum(rows: np.ndarray):
    """A rank's partial sum of its ``[L, n]`` published rows, accumulated in float64 in node order, and its bound: each
    of the L - 1 additions is charged ``U64`` times the magnitude it passes through."""
    s = np.zeros(rows.shape[1])
    mag = np.zeros_like(s)
    for j in range(rows.shape[0]):
        s = s + rows[j]
        mag += np.abs(rows[j])
    return s, max(rows.shape[0] - 1, 0) * U64 * mag


def pga_mix(i, theta_i, pub_rows, nbrs, W, u, *, glob, gossip, sums=None):
    """Node i's mixed row and its bound.  Global: the network sum ``sums = (S, err_S)`` over N nodes divided by N in
    float64 and rounded once to the kernel's dtype (unit ``u``).  Gossip: ``W_ii theta_i + sum_e W_ie pub_e`` in neighbor
    order, every product and sum rounded.  Local SGD: ``theta_i`` unchanged (exact)."""
    if glob:
        N = pub_rows.shape[0]
        m = sums[0] / N
        return m, (u + U64) * np.abs(m) + sums[1] / N
    if not gossip:
        return theta_i.copy(), np.zeros_like(theta_i)
    x = W[i, i] * theta_i
    mag = np.abs(x)
    for j in nbrs[i]:
        t = W[i, j] * pub_rows[j]
        x = x + t
        mag += np.abs(t)
    return x, (len(nbrs[i]) + 2) * u * (mag + np.abs(x))


def dsgd_step(theta, grad_parts, alpha, u):
    """``theta - alpha sum_s g_s`` of one node and its bound (the step launch is DSGD's, unchanged)."""
    S = grad_parts.shape[0]
    g = grad_parts.sum(0)
    eg = max(S - 1, 0) * u * np.abs(grad_parts).sum(0)
    th = theta - alpha * g
    return th, alpha * eg + u * (np.abs(theta) + 2.0 * alpha * np.abs(g))
