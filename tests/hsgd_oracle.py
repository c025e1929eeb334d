"""Float64 NumPy oracle of GT-HSGD (optimizers/gt_hsgd.py), written from the equations, not from consensus_ref.

Round k of every node, with the mixing matrix W_k of the round:

    theta <- W_k (theta - alpha y)
    g  = grad(theta, k);  gp = grad(theta_prev, k)                 (the same minibatch, draw k)
    v' = g (k == 0), g + (1 - beta) (v - gp) otherwise
    y  <- W_k y + v' - v;  v <- v';  theta_prev <- theta

``hsgd_track`` is the tracking step of one round for a kernel launch: the network rows of y, a node's Metropolis row
and its summed partials, with the forward error bound of every output element."""
from __future__ import annotations

import numpy as np


def metropolis(g) -> np.ndarray:
    """W_ij = 1 / (1 + max(d_i, d_j)) on edges, W_ii = 1 - sum_j W_ij."""
    N = g.number_of_nodes()
    d = np.array([g.degree(i) for i in range(N)], dtype=np.float64)
    W = np.zeros((N, N))
    for i, j in g.edges():
        if i != j:
            W[i, j] = W[j, i] = 1.0 / (1.0 + max(d[i], d[j]))
    W[np.diag_indices(N)] = 1.0 - W.sum(1)
    return W


def run(theta0: np.ndarray, Ws, alpha: float, beta: float, grad, rounds: int):
    """Yield ``(theta, y, v, theta_prev)`` after every round; ``grad(x, k)`` is the ``[N, n]`` gradient of every node
    at points ``x`` on draw k, ``Ws[k]`` the round's matrix."""
    theta = np.array(theta0, dtype=np.float64)
    y = np.zeros_like(theta)
    v = np.zeros_like(theta)
    tp = theta.copy()
    omb = 1.0 - beta
    for k in range(rounds):
        W = Ws[k]
        theta = W @ (theta - alpha * y)
        g = grad(theta, k)
        gp = grad(tp, k)
        vn = g if k == 0 else g + omb * (v - gp)
        y = W @ y + vn - v
        v = vn
        tp = theta.copy()
        yield theta.copy(), y.copy(), v.copy(), tp.copy()


def hsgd_track(y_rows, w_self, w_nbr, nbr_rows, g_parts, gp_parts, v, theta, omb, first, u):
    """One node's hsgd_track in float64: ``y_new = w_self y_i + sum_e w_e y_e + (v' - v)``, ``v'``, and the published
    theta.  ``g_parts`` / ``gp_parts`` ``[S, n]`` are the partial rows of the two forward/backward launches.  Returns
    ``(y_new, v_new), (err_y, err_v)``: first-order bounds (in units of the result) of the kernel's rounding, summed
    term by term: every product and sum of a term contributes ``u`` times the magnitude it passes through."""
    S = g_parts.shape[0]
    g = g_parts.sum(0)
    eg = (S - 1) * u * np.abs(g_parts).sum(0)
    if first:
        vn, ev = g, eg
    else:
        gp = gp_parts.sum(0)
        egp = (S - 1) * u * np.abs(gp_parts).sum(0)
        d = v - gp
        vn = g + omb * d
        ev = eg + np.abs(omb) * (egp + u * np.abs(d)) + 2 * u * (np.abs(omb * d) + np.abs(vn))
    ym = w_self * y_rows + sum(w * r for w, r in zip(w_nbr, nbr_rows))
    terms = [np.abs(w_self * y_rows)] + [np.abs(w * r) for w, r in zip(w_nbr, nbr_rows)]
    ey = sum((len(terms) + 1) * u * t for t in terms)
    dv = vn - v
    yn = ym + dv
    ey = ey + ev + u * np.abs(dv) + u * np.abs(yn)
    return (yn, vn), (ey, ev)
