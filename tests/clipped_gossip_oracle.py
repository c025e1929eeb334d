"""Float64 oracle of ClippedGossip (optimizers/clipped_gossip.py), written from the rules: distances, radius, the
self-centred clipped mix, DSGD's step and the attack rows.  Every node of the graph, one round at a time."""
import numpy as np

HONEST, SIGN_FLIP, ALIE = 0, 1, 2
ATTACK = {"sign_flip": SIGN_FLIP, "alie": ALIE}
SLACK = 1e-6        # a prefix of weights fits in delta up to this (fp32 tables round 1/10 up)


def neighbors(W, i):
    return [j for j in range(W.shape[0]) if j != i and W[i, j] != 0.0]


def radius(d, w, delta):
    """(factors, tau, clipped neighbor positions): the neighbors by decreasing distance (ties: the smaller position
    first) are clipped while their weights sum to at most delta; tau is the distance of the first that does not fit."""
    order = sorted(range(len(d)), key=lambda e: (-d[e], e))
    cum, tau, clipped = 0.0, 0.0, []
    for e in order:
        if cum + w[e] > delta + SLACK:
            tau = d[e]
            break
        cum += w[e]
        clipped.append(e)
    f = np.array([tau / d[e] if d[e] > tau else 1.0 for e in range(len(d))])
    return f, tau, clipped


def margins(d, w, delta):
    """Smallest relative gap between two distances of a node, and smallest |prefix weight sum - delta| in the order
    the radius walks: the radius choice is not decided by rounding when both are well above round-off."""
    ds = sorted(d, reverse=True)
    gap = min([abs(a - b) / max(abs(a), abs(b), 1e-300) for a, b in zip(ds, ds[1:])], default=np.inf)
    order = sorted(range(len(d)), key=lambda e: (-d[e], e))
    pre = np.cumsum([w[e] for e in order])
    return gap, min([abs(p - delta - SLACK) for p in pre], default=np.inf)


def mix(theta, pub, W, clip, delta):
    """The round's mix of every node; returns (mixed rows, per-node (neighbors, distances, factors, tau))."""
    N = theta.shape[0]
    out = np.zeros_like(theta)
    info = []
    for i in range(N):
        nb = neighbors(W, i)
        d = np.array([np.linalg.norm(pub[j] - theta[i]) for j in nb])
        w = np.array([W[i, j] for j in nb])
        if clip == "none":
            out[i] = W[i, i] * theta[i] + sum(W[i, j] * pub[j] for j in nb)
            f, tau = np.ones(len(nb)), np.inf
        else:
            f, tau, _ = radius(d, w, delta)
            out[i] = theta[i] + sum(w[e] * f[e] * (pub[j] - theta[i]) for e, j in enumerate(nb))
        info.append((nb, d, f, tau))
    return out, info


def publish(theta, pub, W, attack, byz, scale, z):
    """Rows published after the step: theta (honest), -scale theta (sign flip), or mu - z sigma of the honest
    neighbors' rows of ``pub`` (ALIE; theta without an honest neighbor)."""
    out = theta.copy()
    for i, code in attack.items():
        if code == SIGN_FLIP:
            out[i] = -scale * theta[i]
        elif code == ALIE:
            hon = [j for j in neighbors(W, i) if j not in byz]
            if hon:
                x = np.stack([pub[j] for j in hon])
                out[i] = x.mean(0) - z * x.std(0)
    return out


def round_(theta, pub, W, grad_fn, alpha, clip="adaptive", delta=0.0, attack=None, scale=1.0, z=1.0):
    """One round of every node: (theta, published rows, mix info)."""
    attack = attack or {}
    byz = set(attack)
    mixed, info = mix(theta, pub, W, clip, delta)
    new = np.stack([mixed[i] - alpha * grad_fn(i, mixed[i]) for i in range(theta.shape[0])])
    return new, publish(new, pub, W, attack, byz, scale, z), info
