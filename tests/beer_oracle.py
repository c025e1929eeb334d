"""Float64 oracle of BEER's gossip and step (``beer_mix`` / ``beer_step`` of ``ops/csrc/consensus.cu``), written in NumPy
from the algorithm; it does not call ``ops/consensus_ref.py``.  Code rows are decoded by ``choco_oracle.decode`` (the
layout of ``csrc/consensus.h``), and the encoder's bytes are checked against ``consensus_ref.choco_encode`` by the tests.

Arrays are ``[N, n_pad]`` float64.  Each launch returns its results and first-order error bounds ``e_*`` in the style of
``consensus_oracle.py`` (every rounding charged one unit ``u`` of the kernel's dtype).
"""
from __future__ import annotations

import numpy as np


def _gossip(i, dec, nbrs, W, u, rel_dec):
    """W_ii dec_i + sum_j W_ij dec_j in the kernel's order, and its bound."""
    t = W[i, i] * dec[i]
    mag = np.abs(t)
    for j in nbrs[i]:
        t = t + W[i, j] * dec[j]
        mag += np.abs(W[i, j] * dec[j])
    return t, u * (mag * (1.0 + rel_dec) + np.abs(t))


def mix(theta, h, s_h, v, s_g, dec_h, dec_g, nbrs, W, gamma, alpha, u, rel_dec):
    """One ``beer_mix`` launch: s_h_i += W_ii dec(qh_i) + sum_j W_ij dec(qh_j), the same for s_g with the v-codes, and
    theta_i += gamma (s_h_i - h_i) - alpha v_i.  Returns (theta, s_h, s_g, e_theta, e_s_h, e_s_g)."""
    th, sh, sg = theta.copy(), s_h.copy(), s_g.copy()
    e_th, e_sh, e_sg = np.zeros_like(theta), np.zeros_like(s_h), np.zeros_like(s_g)
    for i in range(theta.shape[0]):
        t, e_t = _gossip(i, dec_h, nbrs, W, u, rel_dec)
        sh[i] = s_h[i] + t
        e_sh[i] = e_t + u * np.abs(sh[i])
        t, e_t = _gossip(i, dec_g, nbrs, W, u, rel_dec)
        sg[i] = s_g[i] + t
        e_sg[i] = e_t + u * np.abs(sg[i])
        d = sh[i] - h[i]
        step = gamma * d - alpha * v[i]
        th[i] = theta[i] + step
        e_th[i] = gamma * (e_sh[i] + u * np.abs(d)) + u * (gamma * np.abs(d) + alpha * np.abs(v[i]) + np.abs(step)
                                                            + np.abs(th[i]))
    return th, sh, sg, e_th, e_sh, e_sg


def step_tracker(v, g, s_g, m_old, grad, e_grad, gamma, u):
    """The tracker update of one ``beer_step`` launch: v + gamma (s_g - g) + grad - m_old (``grad`` the summed partials
    with bound ``e_grad``).  Returns (v, e_v).  The codes and the estimates h += dec(qh), g += dec(qg) are exact given
    the kernel's differences, and are checked against ``consensus_ref.choco_encode`` directly."""
    d = s_g - g
    vn = v + gamma * d + grad - m_old
    e = (e_grad + 2.0 * gamma * u * np.abs(d)
         + 2.0 * u * (np.abs(v) + gamma * np.abs(d) + np.abs(grad) + np.abs(m_old)) + u * np.abs(vn))
    return vn, e
