"""Float64 oracle of K-GT and local DSGD, written from the recursion in ``optimizers/kgt.py`` as plain NumPy loops; it
does not call ``ops/consensus_ref.py``.

``round_`` is one whole round (mix, K gradient steps) for the CPU tests.  ``mix`` and ``step`` are one ``kgt_mix`` and
one ``kgt_step(p)`` launch with the first-order error bound of ``tests/consensus_oracle.py`` (each rounding charged one
unit ``u`` of the kernel's dtype, on the magnitudes of its operands) for the GPU tests."""
from __future__ import annotations

import numpy as np

import consensus_oracle as co


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


def round_(theta, c, y, *, W, grad_fn, alpha, K, correction):
    """One round of every node from the published (theta, y) and the correction c.  Returns (theta, c, y, x, gs): the
    rows after the K steps, the new correction and tracker (None without correction), the mixed rows and the K
    gradients."""
    x = wmix(theta, W)
    if correction:
        c = c + (wmix(y, W) - y)
    th, d, gs = x.copy(), None, []
    for p in range(K):
        g = np.stack([grad_fn(i, th[i]) for i in range(th.shape[0])])
        gs.append(g)
        u = g + c if correction else g
        th = th - alpha * u
        d = u.copy() if p == 0 else d + u
    return th, c, (d / K if correction else None), x, gs


def mix(st, *, k, nbrs, W, u, sum_mode=False, sums=None):
    """One ``kgt_mix`` launch of round k: theta_i <- sum_j W_ij theta_j (own row live, neighbors published) and
    c_i += sum_j W_ij y_j - y_i over the published trackers.  Complete graph: S_theta / N and S_y / N - y_i."""
    out, err = co.dsgd_mix(st, k=k, nbrs=nbrs, W=W, u=u, sum_mode=sum_mode, sums=sums)
    N = st["theta"].shape[0]
    par = k & 1
    yp = st["pub"][par, 1]
    c = st["c"].copy()
    e_c = np.zeros_like(c)
    for i in range(N):
        if sum_mode:
            ym = sums[0][1] / N
            e_ym = sums[1][1] / N
        else:
            ym, e_ym = co._mix(i, yp[i], yp, nbrs, W, u)
        diff = ym - yp[i]
        e_diff = e_ym + u * (np.abs(ym) + np.abs(yp[i]))
        c[i] = st["c"][i] + diff
        e_c[i] = e_diff + u * (np.abs(st["c"][i]) + np.abs(diff) + np.abs(c[i]))
    out["c"], err["c"] = c, e_c
    return out, err


def step(st, *, k, p, K, alpha, correction, u):
    """One ``kgt_step(p)`` launch of round k.  ``u_i = g_i + c_i`` (``g_i`` without correction), theta -= alpha u,
    d = u (p = 0: d is not read) or d + u.  The last step publishes theta and y = d / K into the other parity."""
    par = k & 1
    g, e_g = co.sum_partials(st["grad_part"], u)
    th0 = st["theta"]
    out, err = dict(st), {}
    if correction:
        uu = g + st["c"]
        e_uu = e_g + u * np.abs(uu)
    else:
        uu, e_uu = g, e_g
    th = th0 - alpha * uu
    e_th = alpha * e_uu + u * (np.abs(th0) + 2.0 * alpha * np.abs(uu))
    out["theta"], err["theta"] = th, e_th
    if correction:
        if p == 0:
            d, e_d = uu, e_uu
        else:
            d = st["d"] + uu
            e_d = e_uu + u * (np.abs(st["d"]) + np.abs(uu) + np.abs(d))
    if p == K - 1:
        pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
        pub[par ^ 1, 0], e_pub[par ^ 1, 0] = th, e_th
        if correction:
            pub[par ^ 1, 1] = d / K
            e_pub[par ^ 1, 1] = e_d / K + u * np.abs(d / K)
        out["pub"], err["pub"] = pub, e_pub
    elif correction:
        out["d"], err["d"] = d, e_d
    return out, err
