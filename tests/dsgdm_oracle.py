"""Float64 oracle of DSGD with momentum (local and quasi-global, Nesterov optional), written from the recursion in
``optimizers/dsgdm.py`` as plain NumPy loops; it does not call ``ops/consensus_ref.py``.

``round_`` is one whole round (mix, gradient, step) for the CPU tests.  ``step`` is one ``dsgdm_step`` launch with
the first-order error bound of ``tests/consensus_oracle.py`` (each rounding charged one unit ``u`` of the kernel's
dtype, on the magnitudes of its operands) for the GPU tests."""
from __future__ import annotations

import numpy as np

import consensus_oracle as co


def mix(theta, W):
    """x_i = sum_j W_ij theta_j, own term first, neighbors in index order."""
    N = theta.shape[0]
    x = np.zeros_like(theta)
    for i in range(N):
        x[i] = W[i, i] * theta[i]
        for j in range(N):
            if j != i and W[i, j] != 0.0:
                x[i] = x[i] + W[i, j] * theta[j]
    return x


def momentum(x, g, m, x_prev, *, k, alpha_prev, beta, quasi_global):
    """(the step's momentum, the stored row m or mhat, the new x_prev)."""
    if quasi_global:
        mhat = np.zeros_like(x) if k == 0 else beta * m + (1.0 - beta) * ((x_prev - x) / alpha_prev)
        return beta * mhat + g, mhat, x.copy()
    mom = g.copy() if k == 0 else beta * m + g
    return mom, mom.copy(), None


def round_(theta, m, x_prev, *, k, W, grad_fn, alpha, alpha_prev, beta, quasi_global, nesterov):
    """Round k of every node; returns (theta, m, x_prev, direction)."""
    x = mix(theta, W)
    g = np.stack([grad_fn(i, x[i]) for i in range(x.shape[0])])
    mom, m_new, xp_new = momentum(x, g, m, x_prev, k=k, alpha_prev=alpha_prev, beta=beta, quasi_global=quasi_global)
    d = g + beta * mom if nesterov else mom
    return x - alpha * d, m_new, xp_new, d


def step(st, *, k, alpha, alpha_prev, beta, quasi_global, nesterov, u):
    """One ``dsgdm_step`` launch of round k on the mixed rows ``st["theta"]``; ``beta`` and the alphas as the kernel
    holds them.  Quasi-global: ``d = (x_prev - x) / alpha_prev`` is charged on the magnitudes |x_prev| + |x|, so the
    bound covers the cancellation of the difference however the kernel forms it."""
    par = k & 1
    g, e_g = co.sum_partials(st["grad_part"], u)
    x = st["theta"]
    b, bc = beta, 1.0 - beta                       # the kernel rounds 1 - beta once: charged below
    out = dict(st)
    err = {}
    if k == 0:
        mb, e_mb = np.zeros_like(x), np.zeros_like(x)
    elif quasi_global:
        xp, mh = st["x_prev"], st["m"]
        d = (xp - x) / alpha_prev
        e_d = u * (np.abs(xp) + np.abs(x)) / alpha_prev + u * np.abs(d)
        mb = b * mh + bc * d
        e_mb = bc * e_d + u * (b * np.abs(mh) + 3.0 * bc * np.abs(d) + np.abs(mb))
    else:
        mb, e_mb = st["m"], np.zeros_like(x)
    mom = b * mb + g
    e_mom = b * e_mb + e_g + u * (b * np.abs(mb) + np.abs(g) + np.abs(mom))
    if nesterov:
        dr = g + b * mom
        e_dr = e_g + b * e_mom + u * (np.abs(g) + 2.0 * b * np.abs(mom) + np.abs(dr))
    else:
        dr, e_dr = mom, e_mom
    th = x - alpha * dr
    e_th = alpha * e_dr + u * (np.abs(x) + 2.0 * alpha * np.abs(dr))
    if quasi_global:
        out["m"], err["m"] = mb, e_mb
        out["x_prev"], err["x_prev"] = x.copy(), np.zeros_like(x)
    else:
        out["m"], err["m"] = mom, e_mom
    out["theta"], err["theta"] = th, e_th
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    pub[par ^ 1, 0], e_pub[par ^ 1, 0] = th, e_th
    out["pub"], err["pub"] = pub, e_pub
    return out, err
