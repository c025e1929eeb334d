"""Float64 NumPy oracle of RelaySum (optimizers/relaysum.py), written from the definition without ``consensus_ref``.

State: ``h`` [N, n] (the half-steps, theta between rounds) and ``msg`` {(i, j): row}, the message node i published for
neighbor j at the end of the last round (missing = zero, as before round 0).  ``nbrs`` is the neighbor list of every
node in its order; ``reach(i, k)`` = |{l : d(i, l) <= k}| comes from breadth-first search here."""
import numpy as np


def hop_distances(nbrs):
    N = len(nbrs)
    d = np.full((N, N), -1, dtype=np.int64)
    for s in range(N):
        d[s, s] = 0
        q = [s]
        while q:
            u = q.pop(0)
            for v in nbrs[u]:
                if d[s, v] < 0:
                    d[s, v] = d[s, u] + 1
                    q.append(v)
    return d


def reach(dist, i, k):
    return int(((dist[i] >= 0) & (dist[i] <= k)).sum())


def mix(h, msg, k, nbrs, dist):
    """``r[i]``: the rows node i receives in round k (neighbor order), and ``x``."""
    N = h.shape[0]
    x = np.zeros_like(h)
    r = []
    for i in range(N):
        ri = [msg.get((j, i), np.zeros(h.shape[1])) for j in nbrs[i]]
        s = np.zeros(h.shape[1])
        for q in ri:
            s = s + q
        x[i] = h[i] + (s - (reach(dist, i, k) - 1) * h[i]) / N
        r.append(ri)
    return x, r


def step(x, r, g, alpha, nbrs):
    """``h = x - alpha g`` and the new messages ``m_{i -> j_e} = h + sum_{e' != e} r_e'`` (e' ascending)."""
    h = x - alpha * g
    msg = {}
    for i, nb in enumerate(nbrs):
        for e, j in enumerate(nb):
            m = h[i].copy()
            for f, q in enumerate(r[i]):
                if f != e:
                    m = m + q
            msg[(i, j)] = m
    return h, msg


def round_(h, msg, k, nbrs, dist, grad_fn, alpha):
    x, r = mix(h, msg, k, nbrs, dist)
    g = np.stack([grad_fn(i, x[i]) for i in range(h.shape[0])])
    h, msg = step(x, r, g, alpha, nbrs)
    return h, msg, x


def relayed_counts(nbrs):
    """The paper's relayed count on a tree: ``c_{i->j} = 1 + sum_{l in N(i), l != j} c_{l->i}`` of round k from those of
    round k-1 (all zero before round 0); returns ``R[i][k] - 1 = sum_{j in N(i)} c_{j->i}`` of rounds 0 .. K - 1 for
    K = N + 1."""
    N = len(nbrs)
    c = {(i, j): 0 for i in range(N) for j in nbrs[i]}
    out = np.zeros((N, N + 1), dtype=np.int64)
    for k in range(N + 1):
        for i in range(N):
            out[i, k] = sum(c[(j, i)] for j in nbrs[i])
        c = {(i, j): 1 + sum(c[(l, i)] for l in nbrs[i] if l != j) for i in range(N) for j in nbrs[i]}
    return out
