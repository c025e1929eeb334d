"""Float64 oracle of BRIDGE (optimizers/bridge.py), written from the rules: the coordinate-wise trimmed mean and median
of a node's own row and its neighbors' published rows, DSGD's step and ClippedGossip's attack rows.  Every node of the
graph, one round at a time."""
import numpy as np

from clipped_gossip_oracle import ALIE, ATTACK, HONEST, SIGN_FLIP, neighbors, publish  # noqa: F401


def screen(x, vals, kind, b=0):
    """The screened row of a node with own row ``x`` [n] and neighbor rows ``vals`` [deg, n]: per element, the trimmed
    mean (own value plus sorted positions [b, deg - b), summed in ascending order, over 1 + max(0, deg - 2b)) or the
    median of the own value and the deg values (the mean of the two middle values of an even count)."""
    deg = len(vals)
    s = np.sort(np.asarray(vals, dtype=np.float64).reshape(deg, len(x)), axis=0)
    if kind == "median":
        allv = np.sort(np.vstack([x[None, :], s]), axis=0)
        m = deg // 2
        return allv[m].copy() if deg % 2 == 0 else 0.5 * (allv[m] + allv[m + 1])
    acc = np.array(x, dtype=np.float64)
    for p in range(b, deg - b):
        acc = acc + s[p]
    return acc / (1 + max(0, deg - 2 * b))


def mix(theta, pub, W, kind, b=0):
    """The round's mix of every node (own term: the node's own theta, never its published row)."""
    return np.stack([screen(theta[i], pub[neighbors(W, i)], kind, b) for i in range(theta.shape[0])])


def honest_range(theta, pub, W, i, byz):
    """Element-wise [min, max] of node i's own row and its honest neighbors' published rows."""
    rows = np.vstack([theta[i][None, :]] + [pub[j][None, :] for j in neighbors(W, i) if j not in byz])
    return rows.min(0), rows.max(0)


def guaranteed(W, i, byz, kind, b):
    """The screening guarantee covers honest node i: at most b Byzantine neighbors (trimmed mean), or fewer Byzantine
    than honest values in its set of deg + 1 (median, the own value is honest)."""
    if i in byz:
        return False
    nb = neighbors(W, i)
    f = sum(j in byz for j in nb)
    return f <= b if kind == "trimmed_mean" else f < len(nb) + 1 - f


def round_(theta, pub, W, grad_fn, alpha, kind="trimmed_mean", b=0, attack=None, scale=1.0, z=1.0):
    """One round of every node: (theta, published rows, mixed rows)."""
    attack = attack or {}
    mixed = mix(theta, pub, W, kind, b)
    new = np.stack([mixed[i] - alpha * grad_fn(i, mixed[i]) for i in range(theta.shape[0])])
    return new, publish(new, pub, W, attack, set(attack), scale, z), mixed
