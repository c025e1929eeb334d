"""Float64 NumPy oracle of PowerGossip, one function per launch (pg_mix, pg_step), written from the definition in
``optimizers/powergossip.py`` without calling ``ops/consensus_ref``.  Each returns the values and a round-off bound per
coordinate in the style of ``tests/consensus_oracle.py``: ``|kernel - oracle| <= c err`` with ``u`` the unit
round-off of the kernel's dtype.

Rows are indexed by global node; ``segs`` is the matrix table ``[(offset, m, n, poff, qoff)]`` (``n = 0``: a 1-D tensor
of length m at ``poff`` in the bias block), ``P``/``Q``/``B`` its sizes.  ``pub[i, e]`` is node i's message for its
slot e of the round's phase, ``rs`` the reverse slots (``nbrs[j][rs[i][e]] == i``)."""
import numpy as np


def mix(theta, vec, pub, nbrs, rs, W, gamma, segs, P, Q, phase, u):
    """Returns ``x, err_x, vec', err_vec'``: ``x = h - gamma sum_e W_ie s_ie U_e`` and the next vectors ``d / |d|``
    (unchanged where ``|d| = 0``)."""
    x, vn = theta.copy(), vec.copy()
    ex, ev = np.zeros_like(theta), np.zeros_like(vec)
    base = Q if phase else P
    for i, nb in enumerate(nbrs):
        acc, mag = np.zeros(theta.shape[1]), np.zeros(theta.shape[1])
        for e, j in enumerate(nb):
            s = 1.0 if i < j else -1.0
            own, oth = pub[i, e], pub[j, rs[i][e]]
            d = s * (own - oth)
            dmag = np.abs(own) + np.abs(oth)
            c = W[i, j] * s
            for off, m, n, poff, qoff in segs:
                if n == 0:
                    acc[off: off + m] += c * d[base + poff: base + poff + m]
                    mag[off: off + m] += abs(c) * dmag[base + poff: base + poff + m]
                    continue
                if phase == 0:
                    a, am, b = d[poff: poff + m], dmag[poff: poff + m], vec[i, e, P + qoff: P + qoff + n]
                    acc[off: off + m * n] += c * np.outer(a, b).ravel()
                    mag[off: off + m * n] += abs(c) * np.outer(am, np.abs(b)).ravel()
                    dl, dlm, out = d[poff: poff + m], dmag[poff: poff + m], poff
                else:
                    a, b, bm = vec[i, e, poff: poff + m], d[qoff: qoff + n], dmag[qoff: qoff + n]
                    acc[off: off + m * n] += c * np.outer(a, b).ravel()
                    mag[off: off + m * n] += abs(c) * np.outer(np.abs(a), bm).ravel()
                    dl, dlm, out = d[qoff: qoff + n], dmag[qoff: qoff + n], P + qoff
                nrm = np.sqrt(np.sum(dl * dl))
                if nrm > 0:
                    v = dl / nrm
                    vn[i, e, out: out + len(dl)] = v
                    # the kernel's d carries u |own - oth|-sized errors per element: relative to |d| they move the
                    # direction by about |err d| / |d| (cancellation makes this the dominant term)
                    rel = np.sqrt(np.sum(dlm * dlm)) / nrm
                    ev[i, e, out: out + len(dl)] = u * (dlm / nrm + np.abs(v) * (rel + len(dl)) + 1.0)
        x[i] = theta[i] - gamma * acc
        k = max(1, len(nb))
        ex[i] = u * ((k + 4) * gamma * mag + np.abs(theta[i]) + np.abs(x[i]))
    return x, ex, vn, ev


def step(theta, g, e_g, alpha, vec, pub, nbrs, segs, P, Q, phase, u, chunk=256):
    """Returns ``h, err_h, pub', err_pub'``: ``h = x - alpha g`` and the messages of ``phase`` (that of the next round)
    in ``pub'`` (``[N, dmax, W]``, slots past deg_i and elements past the phase's length unchanged)."""
    h = theta - alpha * g
    eh = alpha * e_g + u * (np.abs(theta) + 2.0 * alpha * np.abs(g))
    out, eo = pub.copy(), np.zeros_like(pub)
    base = Q if phase else P
    for i, nb in enumerate(nbrs):
        for e in range(len(nb)):
            for off, m, n, poff, qoff in segs:
                if n == 0:
                    out[i, e, base + poff: base + poff + m] = h[i, off: off + m]
                    eo[i, e, base + poff: base + poff + m] = eh[i, off: off + m]
                    continue
                H, EH = h[i, off: off + m * n].reshape(m, n), eh[i, off: off + m * n].reshape(m, n)
                if phase == 0:
                    q = vec[i, e, P + qoff: P + qoff + n]
                    out[i, e, poff: poff + m] = H @ q
                    eo[i, e, poff: poff + m] = EH @ np.abs(q) + u * (n + 5) * (np.abs(H) @ np.abs(q))
                else:
                    p = vec[i, e, poff: poff + m]
                    out[i, e, qoff: qoff + n] = p @ H
                    eo[i, e, qoff: qoff + n] = np.abs(p) @ EH + u * (m + 5) * (np.abs(p) @ np.abs(H))
    return h, eh, out, eo
