"""Float64 oracle of DeTAG, written from the recursion in ``optimizers/detag.py`` as plain NumPy loops; it does not call
``ops/consensus_ref.py``.

``weights`` gives the Chebyshev sub-step weights from the closed form ``w_s = 2 mu T_s(mu) / T_{s+1}(mu)``
(``mu = 1 / lam``), not from the recursion the optimizer uses.  ``round_`` is one whole gradient round for the CPU tests.
``gossip`` and ``track`` are one ``ag_gossip(s)`` and one ``detag_track`` launch with the first-order error bound of
``tests/consensus_oracle.py`` (each rounding charged one unit ``u`` of the kernel's dtype, on the magnitudes of its
operands) for the GPU tests."""
from __future__ import annotations

import math

import numpy as np

import consensus_oracle as co


def lam(W):
    """Second largest |eigenvalue| of a symmetric doubly stochastic W (the largest is 1, on the constant vector)."""
    N = W.shape[0]
    if N == 1:
        return 0.0
    ev = np.sort(np.abs(np.linalg.eigvals(np.asarray(W, dtype=np.float64)).real))
    return float(ev[-2])


def cheb_t(n, x):
    """Chebyshev polynomial T_n(x) for x >= 1."""
    return math.cosh(n * math.acosh(x))


def weights(lam_, K, accelerate=True):
    if not accelerate or lam_ == 0.0:
        return [1.0] * K
    mu = 1.0 / lam_
    return [1.0] + [2.0 * mu * cheb_t(s, mu) / cheb_t(s + 1, mu) for s in range(1, K)]


def contraction_bound(lam_, K):
    """Worst-case contraction of the disagreement after K accelerated sub-steps: 1 / T_K(1 / lam)."""
    return 0.0 if lam_ == 0.0 else 1.0 / cheb_t(K, 1.0 / lam_)


def wmix(rows, W):
    """x_i = sum_j W_ij rows_j, own term first, neighbors in index order."""
    N = rows.shape[0]
    x = np.zeros_like(rows)
    for i in range(N):
        x[i] = W[i, i] * rows[i]
        for j in range(N):
            if j != i and W[i, j] != 0.0:
                x[i] = x[i] + W[i, j] * rows[j]
    return x


def gossip_all(X, W, omega):
    """K sub-steps X_{s+1} = X_{s-1} + w_s (W X_s - X_{s-1}) from X_0 = X."""
    x, xp = X, None
    for w in omega:
        m = wmix(x, W)
        xn = m if w == 1.0 else xp + w * (m - xp)
        x, xp = xn, x
    return x


def round_(z, y, g_old, *, W, grad_fn, alpha, omega):
    """One gradient round of every node from the published (z, y).  Returns (theta, y, g, z): the model the gradient was
    taken at, the new tracker, the gradient (the next g_old) and the new published z."""
    theta = gossip_all(z, W, omega)
    ym = gossip_all(y, W, omega)
    g = np.stack([grad_fn(i, theta[i]) for i in range(theta.shape[0])])
    y_new = ym + (g - g_old)
    return theta, y_new, g, theta - alpha * y_new


def gossip(st, *, p, s, K, omega, nbrs, W, u):
    """One ``ag_gossip(s)`` launch of protocol round p on both channels: M = sum_j W_ij X_s,j over the parity p & 1 rows
    (own row included) and X_{s+1} = X_{s-1} + w (M - X_{s-1}), X_{s-1} the own row of parity (p + 1) & 1.  s < K - 1
    writes X_{s+1} into parity (p + 1) & 1; the last sub-step writes theta (channel 0) and ymix (channel 1)."""
    par = p & 1
    pub = st["pub"]
    N = pub.shape[2]
    out, err = dict(st), {}
    res, e_res = np.zeros((2,) + pub.shape[2:]), np.zeros((2,) + pub.shape[2:])
    for ch in range(2):
        rows = pub[par, ch]
        for i in range(N):
            m, e_m = co._mix(i, rows[i], rows, nbrs, W, u)
            if omega == 1.0:
                res[ch, i], e_res[ch, i] = m, e_m
            else:
                xp = pub[par ^ 1, ch, i]
                d = m - xp
                e_d = e_m + u * np.abs(d)
                r = xp + omega * d
                res[ch, i] = r
                e_res[ch, i] = abs(omega) * e_d + u * (np.abs(xp) + 2.0 * abs(omega * d) + np.abs(r))
    if s == K - 1:
        out["theta"], err["theta"] = res[0], e_res[0]
        out["ymix"], err["ymix"] = res[1], e_res[1]
    else:
        pub2, e_pub = pub.copy(), np.zeros_like(pub)
        pub2[par ^ 1, :, :N], e_pub[par ^ 1, :, :N] = res, e_res
        out["pub"], err["pub"] = pub2, e_pub
    return out, err


def track(st, *, p, alpha, u):
    """One ``detag_track`` launch in protocol round p: y = ymix + (g - g_old), g_old = g, publish z = theta - alpha y and
    y into parity (p + 1) & 1."""
    par = p & 1
    g, e_g = co.sum_partials(st["grad_part"], u)
    go = st["g_old"]
    d = g - go
    e_d = e_g + u * np.abs(d)
    y = st["ymix"] + d
    e_y = e_d + u * (np.abs(st["ymix"]) + np.abs(d) + np.abs(y))
    th = st["theta"]
    z = th - alpha * y
    e_z = alpha * e_y + u * (np.abs(th) + 2.0 * alpha * np.abs(y) + np.abs(z))
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    N = th.shape[0]
    pub[par ^ 1, 0, :N], e_pub[par ^ 1, 0, :N] = z, e_z
    pub[par ^ 1, 1, :N], e_pub[par ^ 1, 1, :N] = y, e_y
    return dict(st, g_old=g, pub=pub), {"g_old": e_g, "pub": e_pub}
