"""Float64 NumPy oracle of Push-DIGing (gradient tracking on push-sum gossip), written from the algorithm and independent
of ``ops/consensus_ref.py`` and ``Topology``: the in-neighbors and out-degrees come straight from the networkx graph
(``sgp_oracle.pull_lists``)."""
import numpy as np

from sgp_oracle import pull_lists


def pdg_round(u, w, y, g_old, g, grad_fn, alpha):
    """Round of every node on graph ``g``: mix u - alpha y, y and w with A_ij = 1 / (d_out(j) + 1) over the in-neighbors
    and the node itself, the gradient at theta = u / w, then the tracker update.  Returns (u, w, y, g_new, theta)."""
    ins, outd = pull_lists(g)
    N = u.shape[0]
    un, wn, ys = np.zeros_like(u), np.zeros_like(w), np.zeros_like(y)
    for i in range(N):
        for j in [i] + ins[i]:
            a = 1.0 / (outd[j] + 1.0)
            un[i] += a * (u[j] - alpha * y[j])
            ys[i] += a * y[j]
            wn[i] += a * w[j]
    theta = un / wn[:, None]
    gn = np.stack([grad_fn(i, theta[i]) for i in range(N)])
    return un, wn, ys + gn - g_old, gn, theta
