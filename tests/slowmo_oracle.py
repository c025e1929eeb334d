"""Float64 NumPy oracle of SlowMo's outer update (optimizers/slowmo.py), written from the equations, not from
consensus_ref.  A global round of node i, with xbar the network mean that pga_mix left in theta and gamma = alpha_{k-1}
(alpha0 at k = 0):

    u     <- beta_s u + (a - xbar) / gamma
    a     <- a - alpha_s gamma u
    theta <- a;  m <- 0

The other launches of a SlowMo round (pga_sum, pga_mix, dsgd_step, dsgdm_step) use their existing oracles
(``tests/pga_oracle.py``, ``tests/dsgdm_oracle.py``).  ``run`` is the whole algorithm, for the composed-round tests."""
from __future__ import annotations

import numpy as np

U64 = 2.0 ** -53


def is_global(k: int, period: int) -> bool:
    return k % period == period - 1


def slowmo_outer(xbar, anchor, u, gamma, slow_lr, slow_momentum, unit):
    """The new ``u`` and ``anchor`` (= ``theta``) of one node and their first-order bounds.  The update is evaluated in
    float64, each operation charged ``U64`` times the magnitude it passes through, and each stored row rounded once to
    the kernel's dtype (unit ``unit``).  The anchor is stepped along the unrounded u."""
    d = anchor - xbar
    un = slow_momentum * u + d / gamma
    eu = 3.0 * U64 * (slow_momentum * np.abs(u) + np.abs(d) / gamma)
    step = slow_lr * gamma
    an = anchor - step * un
    ea = unit * np.abs(an) + 3.0 * U64 * (np.abs(anchor) + step * np.abs(un)) + step * eu
    return un, unit * np.abs(un) + eu, an, ea


def run(theta0, Ws, alphas, alpha0, period, gossip, grad, rounds, slow_lr, slow_momentum, base_momentum=0.0,
        nesterov=False):
    """Yield ``(theta, anchor, u)`` after every round; ``grad(x, k)`` is the ``[N, n]`` gradient of every node at points
    ``x`` on draw k, ``Ws[k]`` the round's matrix and ``alphas[k]`` its step."""
    theta = np.array(theta0, dtype=np.float64)
    anchor, u, m = theta.copy(), np.zeros_like(theta), np.zeros_like(theta)
    for k in range(rounds):
        gamma = alpha0 if k == 0 else alphas[k - 1]
        if is_global(k, period):
            xbar = theta.mean(0, keepdims=True)
            u = slow_momentum * u + (anchor - xbar) / gamma
            anchor = anchor - slow_lr * gamma * u
            theta = anchor.copy()
            m = np.zeros_like(m)
        elif gossip:
            theta = Ws[k] @ theta
        g = grad(theta, k)
        if base_momentum > 0.0:
            m = base_momentum * m + g
            theta = theta - alphas[k] * (g + base_momentum * m if nesterov else m)
        else:
            theta = theta - alphas[k] * g
        yield theta.copy(), anchor.copy(), u.copy()
