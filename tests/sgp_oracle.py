"""Float64 NumPy oracle of SGP (push-sum SGD), written from the algorithm and independent of ``ops/consensus_ref.py``
and ``Topology``: the in-neighbors and out-degrees come straight from the networkx graph."""
import numpy as np


def pull_lists(g):
    """(in-neighbors of every node, out-degree of every node); an undirected edge goes both ways."""
    N = g.number_of_nodes()
    if g.is_directed():
        ins = [sorted(int(j) for j in g.predecessors(i) if j != i) for i in range(N)]
        outd = np.array([sum(1 for j in g.successors(i) if j != i) for i in range(N)], dtype=np.float64)
    else:
        ins = [sorted(int(j) for j in g.neighbors(i) if j != i) for i in range(N)]
        outd = np.array([len(n) for n in ins], dtype=np.float64)
    return ins, outd


def column_stochastic(g):
    """A_ij = 1 / (d_out(j) + 1) for j -> i and j = i."""
    ins, outd = pull_lists(g)
    N = len(ins)
    A = np.zeros((N, N))
    for i in range(N):
        A[i, i] = 1.0 / (outd[i] + 1.0)
        for j in ins[i]:
            A[i, j] = 1.0 / (outd[j] + 1.0)
    return A


def mix(x, w, g):
    """One push-sum combine of every node: (x', w', theta' = x' / w')."""
    ins, outd = pull_lists(g)
    xn, wn = np.zeros_like(x), np.zeros_like(w)
    for i in range(x.shape[0]):
        xn[i] = x[i] / (outd[i] + 1.0)
        wn[i] = w[i] / (outd[i] + 1.0)
        for j in ins[i]:
            xn[i] += x[j] / (outd[j] + 1.0)
            wn[i] += w[j] / (outd[j] + 1.0)
    return xn, wn, xn / wn[:, None]


def sgp_round(x, w, g, grad_fn, alpha):
    """Round of every node: mix, gradient at theta = x / w, step on x.  Returns (x, w, theta)."""
    x, w, theta = mix(x, w, g)
    gr = np.stack([grad_fn(i, theta[i]) for i in range(x.shape[0])])
    x = x - alpha * gr
    return x, w, x / w[:, None]
