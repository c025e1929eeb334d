"""Float64 oracle of the consensus kernels in ``ops/csrc/consensus.cu``, one function per launch.

Written from the update equations (``optimizers/{dinno,dsgd,dsgt}.py``, the reference optimizers) as plain per-node,
per-neighbor loops in NumPy float64; it does not call ``ops/consensus_ref.py``, the other thing the kernels are
compared with.  Every function takes the state read back before a launch and returns the state after it, plus, for
every array it writes, a first-order error bound ``err``: the same expression evaluated on absolute values, each
rounding charged one unit ``u`` of the kernel's dtype.  A kernel is right when ``|kernel - oracle| <= c * err``
coordinate by coordinate with ``c`` of order 10 (the number of roundings on the longest path); where ``err`` is 0 the
kernel must be exact.

Inputs use the published-row layout of the kernels: ``pub[par, chan, node, :]``; ``theta``, ``dual`` ... are
``[N, n]``, ``grad_part`` is ``[N, S, n]``.  ``nbrs[i]`` lists node i's neighbors without itself and ``W`` is the
float64 Metropolis matrix.  The complete-graph ("sum") mode reduces in float64 inside the kernel, so its network sum is
charged ``U64`` whatever the dtype.
"""
from __future__ import annotations

import math

import numpy as np

U32, U64 = 2.0 ** -24, 2.0 ** -53
WEIGHT_DECAY = 1e-2


def unit_roundoff(dtype) -> float:
    return U64 if np.dtype(dtype) == np.float64 else U32


def adam_constants(dtype):
    """(beta1, beta2, eps, weight decay) as the kernel of ``dtype`` holds them.  The update is defined with 0.9 / 0.999;
    a float32 kernel can only hold their nearest floats, and ``1 - beta2`` of float32(0.999) is 1.3e-5 away from 1e-3.
    That is representation, not round-off, so the oracle runs with the same constants and the bound measures the
    arithmetic alone."""
    t = np.dtype(dtype).type
    return tuple(float(t(x)) for x in (0.9, 0.999, 1e-8, WEIGHT_DECAY))


# ------------------------------------------------------------------------------------------ schedules ----
def rho_table(conf, oits):
    """rho_k = rho_init * rho_scaling^(k+1): scaled before its first use."""
    return np.array([float(conf["rho_init"]) * float(conf["rho_scaling"]) ** (k + 1) for k in range(oits)])


def lr_table(conf, oits):
    """Primal learning rate of round k: constant, linear or log decay from primal_lr_start to primal_lr_finish; a
    persistent optimizer keeps the first entry unless persistent_follows_schedule."""
    a, kind = float(conf["primal_lr_start"]), conf["lr_decay_type"]
    if kind == "constant":
        t = np.full(oits, a)
    else:
        b = float(conf["primal_lr_finish"])
        x = np.arange(oits) / max(oits - 1, 1)
        t = a + (b - a) * x if kind == "linear" else a * (b / a) ** x
    if conf["persistant_primal_opt"] and not conf.get("persistent_follows_schedule", False):
        t = np.full(oits, t[0])
    return t


def dsgd_alpha_table(alpha0, mu, oits):
    """alpha_k = alpha_{k-1} (1 - mu alpha_{k-1}), starting from alpha0 (the first round already uses the update)."""
    out, a = [], float(alpha0)
    for _ in range(oits):
        a = a * (1.0 - mu * a)
        out.append(a)
    return np.array(out)


# ---------------------------------------------------------------------------------------- building blocks ----
def sum_partials(grad_part, u):
    """The gradient of each node: its S partial rows summed."""
    g = np.zeros(grad_part.shape[::2])
    mag = np.zeros_like(g)
    for i in range(grad_part.shape[0]):
        for s in range(grad_part.shape[1]):
            g[i] += grad_part[i, s]
            mag[i] += np.abs(grad_part[i, s])
    return g, u * mag


def local_sum(pub, par):
    """Complete-graph mode: float64 sum over every node of the published rows of parity ``par``, per channel."""
    s = np.zeros(pub.shape[1:2] + pub.shape[3:])
    mag = np.zeros_like(s)
    for ch in range(pub.shape[1]):
        for j in range(pub.shape[2]):
            s[ch] += pub[par, ch, j]
            mag[ch] += np.abs(pub[par, ch, j])
    return s, U64 * mag


def _mix(i, own, rows, nbrs, W, u):
    """sum_j W_ij x_j with the node's own term from ``own``, neighbors from ``rows``."""
    x = W[i, i] * own
    mag = np.abs(W[i, i] * own)
    for j in nbrs[i]:
        x = x + W[i, j] * rows[j]
        mag += np.abs(W[i, j] * rows[j])
    return x, u * (mag + np.abs(x))


# ---------------------------------------------------------------------------------------------- DiNNO ----
def dinno_update(st, *, step, k, nbrs, rho, lr, opt, pits, persistent, u, dtype, sum_mode=False, sums=None):
    """One ``dinno_update(step)`` launch of round k.

    Step 0 first builds delta_i = sum_j (theta_j^k - theta_i^k) from the published rows (complete graph: the network
    sum minus N theta_i) and takes the dual ascent dual_i -= rho delta_i.  Every step then takes the gradient
    ``g = grad + dual + 2 rho d_i (theta - theta_i^k) - rho delta_i`` and one SGD / Adam / AdamW step with bias
    correction at t = k pits + step + 1 (persistent moments) or step + 1 (moments reset every round).  The last
    step publishes theta into the other parity."""
    N = st["theta"].shape[0]
    par = k & 1
    out = {key: (v.copy() if isinstance(v, np.ndarray) else v) for key, v in st.items()}
    err = {key: np.zeros_like(v) for key, v in st.items() if v is not None and key in ("theta", "dual", "delta", "m", "v")}
    err["pub"] = np.zeros_like(st["pub"])
    gl, e_gl = sum_partials(st["grad_part"], u)
    b1, b2, eps, wd = adam_constants(dtype)
    t = k * pits + step + 1 if persistent else step + 1
    for i in range(N):
        th = st["theta"][i]
        d = len(nbrs[i])
        if step == 0:
            thk = th
            if sum_mode:
                dl = sums[0][0] - N * thk
                e_dl = u * np.abs(dl) + U64 * N * np.abs(thk) + sums[1][0]
            else:
                dl = np.zeros_like(th)
                mag = np.zeros_like(th)
                for j in nbrs[i]:
                    diff = st["pub"][par, 0, j] - thk
                    dl = dl + diff
                    mag += np.abs(diff)
                e_dl = u * mag
            du = st["dual"][i] - rho * dl
            e_du = u * (np.abs(st["dual"][i]) + rho * np.abs(dl)) + rho * e_dl
            out["delta"][i], err["delta"][i] = dl, e_dl
            out["dual"][i], err["dual"][i] = du, e_du
        else:
            thk = st["pub"][par, 0, i]
            dl, du = st["delta"][i], st["dual"][i]
            e_dl = e_du = np.zeros_like(th)
        g = gl[i] + du + 2.0 * rho * d * (th - thk) - rho * dl
        e_g = (e_gl[i] + e_du + rho * e_dl
               + u * (np.abs(gl[i]) + np.abs(du) + 4.0 * rho * d * np.abs(th - thk) + rho * np.abs(dl) + np.abs(g)))
        if opt == "sgd":
            new = th - lr * g
            e_new = u * (np.abs(th) + 2.0 * lr * np.abs(g)) + lr * e_g
        else:
            fresh = step == 0 and not persistent
            m0 = np.zeros_like(th) if fresh else st["m"][i]
            v0 = np.zeros_like(th) if fresh else st["v"][i]
            m = b1 * m0 + (1.0 - b1) * g
            e_m = u * (b1 * np.abs(m0) + (1.0 - b1) * np.abs(g) + np.abs(m)) + (1.0 - b1) * e_g
            v = b2 * v0 + (1.0 - b2) * g * g
            e_v = u * (b2 * v0 + 2.0 * (1.0 - b2) * g * g + v) + (1.0 - b2) * 2.0 * np.abs(g) * e_g
            step_v, e_step = adam_step(m, v, e_m, e_v, lr=lr, t=t, u=u, b1=b1, b2=b2, eps=eps)
            base, e_base = th, np.zeros_like(th)
            if opt == "adamw":
                base = th * (1.0 - lr * wd)
                e_base = 2.0 * u * np.abs(th)
            new = base - step_v
            e_new = e_base + e_step + u * (np.abs(base) + np.abs(step_v))
            out["m"][i], err["m"][i] = m, e_m
            out["v"][i], err["v"][i] = v, e_v
        out["theta"][i], err["theta"][i] = new, e_new
        if step == pits - 1:
            out["pub"][par ^ 1, 0, i], err["pub"][par ^ 1, 0, i] = new, e_new
    return out, err


def adam_step(m, v, e_m, e_v, *, lr, t, u, b1, b2, eps):
    """The Adam step ``lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps)`` and its bound, carried through from the bounds on
    m and v.  The bias corrections 1 - beta^t are computed in the kernel's dtype: their magnitude 1 + t beta^t over
    their value is the condition number that turns one rounding of beta^t into the relative error of the step."""
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    rel_s = u * (2.0 + (1.0 + t * b1 ** t) / bc1)
    bs = math.sqrt(bc2)
    rel_b = u * (1.0 + 0.5 * (1.0 + t * b2 ** t) / bc2)
    s = lr / bc1
    sv = np.sqrt(v)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_sv = np.where(sv > 0, np.minimum(e_v / (2.0 * sv), np.sqrt(e_v)), np.sqrt(e_v)) + u * sv
    D = sv / bs + eps
    e_D = e_sv / bs + (sv / bs) * rel_b + u * D
    step = s * m / D
    e_step = np.abs(step) * (rel_s + 2.0 * u) + s * e_m / D + s * np.abs(m) * e_D / (D * D)
    return step, e_step


# ----------------------------------------------------------------------------------------------- DSGD ----
def dsgd_mix(st, *, k, nbrs, W, u, sum_mode=False, sums=None):
    """theta_i <- sum_j W_ij theta_j^k (own row live, neighbors published); complete graph: the network mean."""
    N = st["theta"].shape[0]
    par = k & 1
    out = dict(st, theta=st["theta"].copy())
    err = {"theta": np.zeros_like(st["theta"])}
    for i in range(N):
        if sum_mode:
            out["theta"][i] = sums[0][0] / N
            err["theta"][i] = u * np.abs(out["theta"][i]) + sums[1][0] / N
        else:
            out["theta"][i], err["theta"][i] = _mix(i, st["theta"][i], st["pub"][par, 0], nbrs, W, u)
    return out, err


def dsgd_step(st, *, k, alpha, u):
    """theta_i -= alpha_k g_i, published into the other parity."""
    par = k & 1
    g, e_g = sum_partials(st["grad_part"], u)
    th = st["theta"] - alpha * g
    e = alpha * e_g + u * (np.abs(st["theta"]) + 2.0 * alpha * np.abs(g))
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    pub[par ^ 1, 0], e_pub[par ^ 1, 0] = th, e
    return dict(st, theta=th, pub=pub), {"theta": e, "pub": e_pub}


# ----------------------------------------------------------------------------------------------- DSGT ----
def dsgt_init(st, *, u):
    """y = g_old = the first gradient; y is published into parity 0."""
    g, e_g = sum_partials(st["grad_part"], u)
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    pub[0, 1], e_pub[0, 1] = g, e_g
    return dict(st, g_old=g, pub=pub), {"g_old": e_g, "pub": e_pub}


def dsgt_mix(st, *, k, nbrs, W, alpha, u, sum_mode=False, sums=None):
    """theta_i <- sum_j W_ij (theta_j - alpha y_j); complete graph: (S_theta - alpha S_y) / N."""
    N = st["theta"].shape[0]
    par = k & 1
    out = dict(st, theta=st["theta"].copy())
    err = {"theta": np.zeros_like(st["theta"])}
    for i in range(N):
        if sum_mode:
            x = (sums[0][0] - alpha * sums[0][1]) / N
            out["theta"][i] = x
            err["theta"][i] = u * np.abs(x) + (sums[1][0] + alpha * sums[1][1]) / N
            continue
        y = st["pub"][par, 1]
        z_own = st["theta"][i] - alpha * y[i]
        x = W[i, i] * z_own
        mag = W[i, i] * (np.abs(st["theta"][i]) + alpha * np.abs(y[i]))
        for j in nbrs[i]:
            x = x + W[i, j] * (st["pub"][par, 0, j] - alpha * y[j])
            mag += W[i, j] * (np.abs(st["pub"][par, 0, j]) + alpha * np.abs(y[j]))
        out["theta"][i], err["theta"][i] = x, u * (2.0 * mag + np.abs(x))
    return out, err


def dsgt_track(st, *, k, nbrs, W, u, sum_mode=False, sums=None):
    """y_i <- sum_j W_ij y_j + g_i^new - g_i^old; g_old <- g^new; y and theta published into the other parity."""
    N = st["theta"].shape[0]
    par = k & 1
    g, e_g = sum_partials(st["grad_part"], u)
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    for i in range(N):
        if sum_mode:
            y = sums[0][1] / N
            e_y = u * np.abs(y) + sums[1][1] / N
        else:
            y, e_y = _mix(i, st["pub"][par, 1, i], st["pub"][par, 1], nbrs, W, u)
        yn = y + g[i] - st["g_old"][i]
        pub[par ^ 1, 1, i] = yn
        e_pub[par ^ 1, 1, i] = e_y + e_g[i] + u * (np.abs(y) + np.abs(g[i]) + np.abs(st["g_old"][i]) + np.abs(yn))
        pub[par ^ 1, 0, i] = st["theta"][i]
    return dict(st, g_old=g, pub=pub), {"g_old": e_g, "pub": e_pub}


# ---------------------------------------------------------------------------------------------- metric ----
def consensus_metric(rows):
    """Distances between L2-normalised rows [N, n]: pairwise [N, N] and to the mean of the normalised rows [N].
    The kernel reads the rows in their dtype and accumulates in float64; the bound charges U64 per term of its
    longest accumulation chain (the per-thread strided loop plus the block reduction)."""
    N, n = rows.shape
    nrm = np.array([max(math.sqrt(float(np.sum(r * r))), 1e-12) for r in rows])
    a = rows / nrm[:, None]
    depth = -(-n // 256) + 16 + N
    pair = np.zeros((N, N))
    e_pair = np.zeros((N, N))
    for i in range(N):
        for j in range(N):
            pair[i, j] = math.sqrt(float(np.sum((a[i] - a[j]) ** 2)))
            e_pair[i, j] = U64 * depth * math.sqrt(float(np.sum((np.abs(a[i]) + np.abs(a[j])) ** 2)))
    mu = a.mean(0)
    mean = np.array([math.sqrt(float(np.sum((a[i] - mu) ** 2))) for i in range(N)])
    e_mean = np.array([U64 * depth * math.sqrt(float(np.sum((np.abs(a[i]) + np.abs(a).mean(0)) ** 2)))
                       for i in range(N)])
    return (pair, e_pair), (mean, e_mean)


def check(name, got, want, err, c):
    """Largest ratio |got - want| / (c err) over the coordinates; raises with the first offending coordinate when
    any exceeds 1 (where err is 0 the values must be equal)."""
    got = np.asarray(got, dtype=np.float64)
    diff = np.abs(got - want)
    bound = c * err
    bad = diff > bound
    if bad.any():
        idx = np.unravel_index(np.argmax(np.where(bad, diff - bound, -np.inf)), diff.shape)
        raise AssertionError(f"{name}: {int(bad.sum())} coordinate(s) outside c*err, first at {idx}: got {got[idx]!r}, "
                             f"oracle {want[idx]!r}, |diff| {diff[idx]:.3e} > bound {bound[idx]:.3e}")
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, diff / bound, 0.0)
    return float(r.max()) if r.size else 0.0
