"""Float64 NumPy oracle of DP-DSGD / DECOR (optimizers/dp_dsgd.py), written from the update rule, and the per-launch
oracles of ``dp_norm`` and ``dp_step``.  The noise rows come from the host twin of the stream
(``ops/consensus_ref.py: dp_noise``), which is the stream's definition; everything else is recomputed here."""
import math

import networkx as nx
import numpy as np

from nn_distributed_training_b200.ops import consensus_ref as ref


def clip_factor(g: np.ndarray, C: float) -> float:
    n = math.sqrt(float(np.dot(g, g)))
    return 1.0 if n <= C else C / n


def noise(key, k, i, nbrs, n_pad, C, z_dp, z_pair, live):
    return ref.dp_noise(key, k, i, list(nbrs), n_pad, C * z_dp, C * z_pair, live)


def run(theta0, graphs, alphas, C, z_dp, z_pair, key, grad, R, live):
    """``theta`` of the N nodes after each of R rounds (``[N, n_pad]`` rows; ``grad(x, k)`` gives the gradients of
    every node at points x on its draw k)."""
    th = np.array(theta0, dtype=np.float64)
    N, n_pad = th.shape
    out = []
    for k in range(R):
        g = graphs[k]
        W = np.zeros((N, N))
        d = np.array([g.degree(i) for i in range(N)], dtype=np.float64)
        for i, j in g.edges():
            if i != j:
                W[i, j] = W[j, i] = 1.0 / (1.0 + max(d[i], d[j]))
        W[np.diag_indices(N)] = 1.0 - W.sum(1)
        x = W @ th
        G = grad(x, k)
        for i in range(N):
            v = noise(key, k, i, sorted(nx.neighbors(g, i)), n_pad, C, z_dp, z_pair, live)
            x[i] = x[i] - alphas[k] * (clip_factor(G[i], C) * G[i] + v)
        th = x
        out.append(th.copy())
    return out


def cycle_inverse_diagonal(N: int, z_dp: float, z_pair: float) -> float:
    """``[Sigma^-1]_ii`` on the N-cycle from the circulant's eigenvalues ``z_dp^2 + z_pair^2 (2 - 2 cos(2 pi m / N))``."""
    m = np.arange(N)
    return float(np.mean(1.0 / (z_dp ** 2 + z_pair ** 2 * (2.0 - 2.0 * np.cos(2.0 * np.pi * m / N)))))


def complete_inverse_diagonal(N: int, z_dp: float, z_pair: float) -> float:
    """``[Sigma^-1]_ii`` on the complete graph: ``(1 - 1/N) / (z_dp^2 + N z_pair^2) + 1 / (N z_dp^2)``."""
    return (1.0 - 1.0 / N) / (z_dp ** 2 + N * z_pair ** 2) + 1.0 / (N * z_dp ** 2)
