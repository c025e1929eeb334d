"""Float64 oracle of decentralized AMSGrad / AdaGrad with and without the gossiped second moment, written from the
recursion in ``optimizers/dadaptive.py`` as plain NumPy; it does not call ``ops/consensus_ref.py``.

``round_`` is one whole round (mix, gradient, step) for the CPU tests.  ``mix`` and ``step`` are one
``dadaptive_mix`` (or ``dsgd_mix``) and one ``dadaptive_step`` launch with the first-order error bound of
``tests/consensus_oracle.py`` (each rounding charged one unit ``u`` of the kernel's dtype, on the magnitudes of its
operands) for the GPU tests."""
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


def init_state(N, n, eps, variant, tracking):
    """m = 0, v = 0 (amsgrad), vhat = eps and the published tracker u~ = eps (tracking)."""
    return {"m": np.zeros((N, n)), "v": np.zeros((N, n)) if variant == "amsgrad" else None,
            "vhat": np.full((N, n), eps), "ut": np.full((N, n), eps) if tracking else None}


def update(g, m, v, vhat, z, *, k, alpha, beta1, beta2, eps, variant):
    """The step of round k given the gradients, the state and z (``None``: own second moment).  Returns the step
    ``alpha m / sqrt(u)`` and the new (m, v, vhat, u~)."""
    m = beta1 * m + (1.0 - beta1) * g
    if variant == "adagrad":
        vn = vhat + (g * g - vhat) / (k + 1)
    else:
        v = beta2 * v + (1.0 - beta2) * g * g
        vn = np.maximum(vhat, v)
    ut = None
    if z is not None:
        ut = z + (vn - vhat)
        u = np.maximum(ut, eps)
    else:
        u = np.maximum(vn, eps)
    return alpha * (m / np.sqrt(u)), m, v, vn, ut


def round_(theta, st, *, k, W, grad_fn, alpha, beta1=0.9, beta2=0.999, eps=1e-8, variant, tracking):
    """One round of every node from the published theta and u~.  Returns (theta, state)."""
    x = wmix(theta, W)
    z = wmix(st["ut"], W) if tracking else None
    g = np.stack([grad_fn(i, x[i]) for i in range(x.shape[0])])
    step, m, v, vhat, ut = update(g, st["m"], st["v"], st["vhat"], z, k=k, alpha=alpha, beta1=beta1, beta2=beta2,
                                  eps=eps, variant=variant)
    return x - step, {"m": m, "v": v, "vhat": vhat, "ut": ut}


# ------------------------------------------------------------------------------------- one launch, bounded ----
def mix(st, *, k, nbrs, W, u, sum_mode=False, sums=None):
    """One ``dadaptive_mix`` launch of round k: x_i = sum_j W_ij theta_j into theta (own row live, neighbors
    published) and z_i = sum_j W_ij u~_j into ut (own and neighbor rows published).  Complete graph: S / N."""
    out, err = co.dsgd_mix(st, k=k, nbrs=nbrs, W=W, u=u, sum_mode=sum_mode, sums=sums)
    N = st["theta"].shape[0]
    up = st["pub"][k & 1, 1]
    z, e_z = np.zeros_like(st["ut"]), np.zeros_like(st["ut"])
    for i in range(N):
        if sum_mode:
            z[i] = sums[0][1] / N
            e_z[i] = u * np.abs(z[i]) + sums[1][1] / N
        else:
            z[i], e_z[i] = co._mix(i, up[i], up, nbrs, W, u)
    out["ut"], err["ut"] = z, e_z
    return out, err


def step(st, *, k, alpha, beta1, beta2, eps, variant, tracking, u):
    """One ``dadaptive_step`` launch of round k on the mixed rows (``st["ut"]`` holds z with tracking).  Writes m,
    v (amsgrad), vhat, theta and publishes theta and u~ into the other parity; ut is left holding z."""
    g, e_g = co.sum_partials(st["grad_part"], u)
    x, m0, vh = st["theta"], st["m"], st["vhat"]
    b1c, b2c = 1.0 - beta1, 1.0 - beta2
    out, err = dict(st), {}
    m = beta1 * m0 + b1c * g
    e_m = b1c * e_g + u * (beta1 * np.abs(m0) + b1c * np.abs(g) + np.abs(m))
    g2 = g * g
    e_g2 = 2.0 * np.abs(g) * e_g + u * g2
    if variant == "adagrad":
        d = g2 - vh
        q = d / (k + 1)
        e_q = (e_g2 + u * np.abs(d)) / (k + 1) + u * np.abs(q)
        vn = vh + q
        e_vn = e_q + u * np.abs(vn)
    else:
        v0 = st["v"]
        v = beta2 * v0 + b2c * g2
        e_v = b2c * e_g2 + u * (beta2 * np.abs(v0) + b2c * g2 + np.abs(v))
        vn = np.maximum(vh, v)
        e_vn = e_v                      # max is 1-Lipschitz and vhat enters exactly
        out["v"], err["v"] = v, e_v
    if tracking:
        dl = vn - vh
        ut = st["ut"] + dl
        e_uu = e_vn + u * np.abs(dl) + u * np.abs(ut)
        uu = np.maximum(ut, eps)
    else:
        uu, e_uu = np.maximum(vn, eps), e_vn
    s = np.sqrt(uu)
    e_s = e_uu / (2.0 * s) + u * s
    q = m / s
    e_q = e_m / s + np.abs(m) * e_s / (s * s) + u * np.abs(q)
    th = x - alpha * q
    e_th = alpha * e_q + u * (np.abs(x) + 2.0 * alpha * np.abs(q))
    out["m"], err["m"] = m, e_m
    out["vhat"], err["vhat"] = vn, e_vn
    out["theta"], err["theta"] = th, e_th
    par = k & 1
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    pub[par ^ 1, 0], e_pub[par ^ 1, 0] = th, e_th
    if tracking:
        pub[par ^ 1, 1], e_pub[par ^ 1, 1] = ut, e_uu
    out["pub"], err["pub"] = pub, e_pub
    return out, err
