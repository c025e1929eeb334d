"""Float64 NumPy oracle of Moniqua (optimizers/moniqua.py), one function per fused launch, written from the paper's
equations (DESIGN §2.17) independently of ops/consensus_ref.py; only the Philox4x32-10 twin is shared.  Each launch
function returns the float64 result, a round-off bound on how far a correct kernel in the arena dtype may be from it,
and (the mix) the margin hits."""
import numpy as np

from nn_distributed_training_b200.ops.consensus_ref import MQ_TAG, philox4x32_10

EPS64 = np.finfo(np.float64).eps


def delta(bits):
    return 2.0 ** -bits


def modulus(theta_bound, bits):
    return 2.0 * theta_bound / (1.0 - 2.0 * delta(bits))


def uniforms(key, k, node, n):
    p = np.arange(n // 4, dtype=np.uint64)
    ctr = np.stack([p, np.full_like(p, k), np.full_like(p, node), np.full_like(p, MQ_TAG)], axis=-1)
    return philox4x32_10(ctr, key).reshape(-1).astype(np.float64) / 2.0 ** 32


def encode(x, B, bits, u, live):
    """Codes (int64) of the float64 values ``x`` with the uniforms ``u``: stochastic rounding of frac(x / B) 2^bits."""
    L = 1 << bits
    z = np.asarray(x, dtype=np.float64) / B
    t = (z - np.floor(z)) * L
    fl = np.floor(t)
    c = (fl.astype(np.int64) + (u < t - fl)) % L
    return np.where(live, c, 0)


def decode(c, y, B, bits):
    """``(xhat, offset)``: the representative of code c nearest to the side information y, and y / B minus it."""
    cl = np.asarray(c, dtype=np.float64) * delta(bits)
    v = np.asarray(y, dtype=np.float64) / B - cl
    n = np.rint(v)
    return B * (cl + n), v - n


def pack(c, bits):
    per = 32 // bits
    w = (c.reshape(-1, per).astype(np.uint64) << (np.arange(per, dtype=np.uint64) * np.uint64(bits))).sum(-1)
    return w.astype(np.uint32).view(np.uint8)


def mix(theta, codes, w_rows, nbrs, lo, B, bits, eps):
    """mq_mix of the local rows ``theta [L, n]`` (float64 of the arena values) on every node's codes ``codes [N, n]``:
    the mixed rows, the bound and the margin hits per node.  The fp64 sum costs a few eps64 of ``|y| + sum |w| |d|``,
    the final rounding half an ulp of the arena dtype (``eps``)."""
    out = np.empty_like(theta)
    bound = np.empty_like(theta)
    hits = np.zeros(theta.shape[0], dtype=np.int64)
    lim = 0.5 - delta(bits)
    for l in range(theta.shape[0]):
        y = theta[l]
        xi, _ = decode(codes[lo + l], y, B, bits)
        acc = np.zeros_like(y)
        mag = np.abs(y)
        for j in nbrs[l]:
            xj, off = decode(codes[j], y, B, bits)
            acc += w_rows[l][j] * (xj - xi)
            mag = mag + abs(w_rows[l][j]) * (np.abs(xj) + np.abs(xi))
            hits[l] += int((np.abs(off) > lim).sum())
        out[l] = y + acc
        bound[l] = 0.5 * eps * np.abs(out[l]) + 8 * (len(nbrs[l]) + 2) * EPS64 * (mag + B)
    return out, bound, hits


def step(theta, psi, g, alpha, first, eps):
    """mq_step's arithmetic on the mixed rows: DSGD's ``theta - alpha g`` (psi None) or Exact Diffusion's adapt /
    correct; returns (theta, psi, bound).  Each operation in the arena dtype rounds once."""
    if psi is None:
        new = theta - alpha * g
        return new, None, 2 * eps * (np.abs(theta) + np.abs(alpha * g))
    psi0 = theta if first else psi
    pn = theta - alpha * g
    new = pn + (theta - psi0)
    bound = 4 * eps * (np.abs(theta) + np.abs(alpha * g) + np.abs(psi0))
    return new, pn, bound


def run(theta0, Ws, alpha0, mu, grad_fn, R, bits, theta_bound, key, base, live):
    """R rounds from ``theta0 [N, n]`` on the mixing matrices ``Ws`` in float64 with ``grad_fn(x, k)``: the rows after
    every round and the margin hits so far."""
    B = modulus(theta_bound, bits)
    N, n = theta0.shape
    theta = theta0.copy()
    psi = np.zeros_like(theta) if base == "exact_diffusion" else None
    codes = np.stack([encode(theta[i], B, bits, uniforms(key, 0, i, n), live) for i in range(N)])
    hits = np.zeros(N, dtype=np.int64)
    alpha = alpha0
    out = []
    for k in range(R):
        W = Ws[k]
        if base == "exact_diffusion":
            W = 0.5 * (np.eye(N) + W)
        nbrs = [[j for j in range(N) if j != i and Ws[k][i, j] != 0] for i in range(N)]
        theta, _, h = mix(theta, codes, W, nbrs, 0, B, bits, EPS64)
        hits += h
        alpha = alpha * (1.0 - mu * alpha)
        g = grad_fn(theta, k)
        if base == "exact_diffusion":
            theta, psi, _ = step(theta, psi, g, alpha, k == 0, EPS64)
        else:
            theta, _, _ = step(theta, None, g, alpha, k == 0, EPS64)
        codes = np.stack([encode(theta[i], B, bits, uniforms(key, k + 1, i, n), live) for i in range(N)])
        out.append((theta.copy(), hits.copy()))
    return out
