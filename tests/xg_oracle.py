"""Float64 NumPy oracle of cross-gradient gossip (optimizers/cross_gradient.py), written from the equations, not from
consensus_ref.

Round k of every node i with neighbours N_i, lam = cross_weight:

    xmix_i = sum_j W_ij x_j
    d_i    = ((1 - lam) + lam W_ii) grad f_i(x_i; k) + sum_{j in N_i} lam W_ij grad f_j(x_i; k)
    x_i   <- xmix_i - alpha_k d_i

``grad(x, k)`` is the ``[N, n]`` gradient of every node's loss at points ``x`` (row j at node j's own point) on its draw
k; node j's gradient at node i's row is row j of ``grad`` evaluated with every row set to ``x_i``.  The per-launch
helpers give each output of one kernel launch with a first-order bound of the kernel's rounding, in the style of
``consensus_oracle.py``."""
from __future__ import annotations

import numpy as np


def run(theta0: np.ndarray, W: np.ndarray, lam: float, alphas, grad, rounds: int):
    """Yield ``theta`` after every round."""
    theta = np.array(theta0, dtype=np.float64)
    N = theta.shape[0]
    nbrs = [[j for j in range(N) if j != i and W[i, j] != 0.0] for i in range(N)]
    for k in range(rounds):
        xmix = W @ theta
        own = grad(theta, k)
        d = np.zeros_like(theta)
        for i in range(N):
            at_i = grad(np.repeat(theta[i: i + 1], N, axis=0), k)
            d[i] = ((1.0 - lam) + lam * W[i, i]) * own[i] + sum(lam * W[i, j] * at_i[j] for j in nbrs[i])
        theta = xmix - alphas[k] * d
        yield theta.copy()


def fixed_point(H, r, W, lam, alpha):
    """Fixed point of the full-batch map ``x <- W x - alpha d(x)`` for quadratic losses with ``grad f_i(x) = H_i x -
    r_i`` (``H [N, n, n]``, ``r [N, n]``): ``d_i(x) = M_i x_i - s_i`` is affine, so ``(I - W (x) I + alpha diag(M)) x =
    alpha s``.  Returns ``[N, n]``."""
    N, n = r.shape
    A = np.eye(N * n) - np.kron(W, np.eye(n))
    s = np.zeros(N * n)
    for i in range(N):
        c0 = (1.0 - lam) + lam * W[i, i]
        M = c0 * H[i] + sum(lam * W[i, j] * H[j] for j in range(N) if j != i)
        A[i * n:(i + 1) * n, i * n:(i + 1) * n] += alpha * M
        s[i * n:(i + 1) * n] = alpha * (c0 * r[i] + sum(lam * W[i, j] * r[j] for j in range(N) if j != i))
    return np.linalg.solve(A, s).reshape(N, n)


def partial_sum(parts, u):
    """``parts [S, n]`` summed in order s = 0, 1, ...; the bound of that sum's rounding."""
    S = parts.shape[0]
    return parts.sum(0), (S - 1) * u * np.abs(parts).sum(0)


def mix(own, w_self, w_nbr, nbr_rows, u):
    """``w_self own + sum_e w_e row_e`` (dsgd_mix) and its bound."""
    terms = [w_self * own] + [w * r for w, r in zip(w_nbr, nbr_rows)]
    return sum(terms), sum((len(terms) + 1) * u * np.abs(t) for t in terms)


def step(xmix, g, coef0, coefs, recv, alpha, u):
    """``xmix - alpha (T)(coef0 g + sum_e coef_e recv_e)`` with d in float64: the bound of the float64 sum, of rounding d
    once to T and of the step."""
    terms = [coef0 * g] + [c * r for c, r in zip(coefs, recv)]
    d = sum(terms)
    x = xmix - alpha * d
    e64 = (len(terms) + 1) * 2.0 ** -53 * sum(np.abs(t) for t in terms)    # the float64 sum, cancellation included
    return x, abs(alpha) * e64 + 2 * u * np.abs(alpha * d) + u * np.abs(x)
