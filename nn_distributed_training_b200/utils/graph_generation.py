"""Communication topologies and mixing matrices.

API parity with the reference ``utils/graph_generation.py`` (same function
names, arguments and return types: ``generate_from_conf`` :69, ``get_metropolis``
:107, ``euclidean_disk_graph`` :125, ``disk_with_fied`` :14, ``gen_delaunay``
:149, ``fied_from_disk`` :9) but implemented on dense adjacency matrices:

* the Metropolis matrix is a closed form over the degree vector (the reference
  runs an O(N^2) Python loop over a scipy Laplacian every round),
* the Fiedler value used by ``disk_with_fied`` comes from a dense symmetric
  eigensolve (N <= a few hundred), so the radius bisection is deterministic for
  a given point set,
* ``Topology`` caches neighbor lists / Metropolis rows and exports the padded
  neighbor table consumed by the fused consensus kernels.
"""
from __future__ import annotations

import random
from typing import Dict, List, Sequence, Tuple

import networkx as nx
import numpy as np
import torch


# --------------------------------------------------------------------------
# dense helpers
# --------------------------------------------------------------------------
def adjacency(graph: nx.Graph) -> np.ndarray:
    """Boolean adjacency [N, N] with nodes taken in ``range(N)`` order and the
    diagonal cleared (self loops never carry a mixing weight).  An undirected
    graph gives a symmetric matrix; a ``DiGraph`` keeps its direction
    (``adj[u, v]`` for the edge ``u -> v``)."""
    n = graph.number_of_nodes()
    adj = np.zeros((n, n), dtype=bool)
    if graph.number_of_edges():
        e = np.asarray(list(graph.edges()), dtype=np.int64)
        adj[e[:, 0], e[:, 1]] = True
        if not graph.is_directed():
            adj[e[:, 1], e[:, 0]] = True
    np.fill_diagonal(adj, False)
    return adj


def push_weights_from_adjacency(adj: np.ndarray) -> np.ndarray:
    """Column-stochastic push-sum matrix (float64): ``A_ij = 1 / (d_out(j) + 1)``
    for every edge ``j -> i`` and for ``i = j``.  Each node sets its column from
    its own out-degree, so no node needs to know anything about the others."""
    adj = np.asarray(adj, dtype=bool)
    inv = 1.0 / (adj.sum(1).astype(np.float64) + 1.0)      # per sender j: 1 / (d_out(j) + 1)
    a = np.where(adj.T, inv[None, :], 0.0)
    a[np.diag_indices_from(a)] = inv
    return a


def is_strongly_connected_adj(adj: np.ndarray) -> bool:
    """Every node reaches every other along the edges' direction."""
    return is_connected_adj(adj) and is_connected_adj(np.asarray(adj).T)


def metropolis_from_adjacency(adj: np.ndarray, degs: np.ndarray | None = None) -> np.ndarray:
    """W_ij = 1/(max(d_i,d_j)+1) on edges, W_ii = 1 - sum_j W_ij (float64)."""
    adj = np.asarray(adj, dtype=bool)
    if degs is None:
        degs = adj.sum(1)
    degs = np.asarray(degs, dtype=np.float64)
    w = np.where(adj, 1.0 / (np.maximum(degs[:, None], degs[None, :]) + 1.0), 0.0)
    w[np.diag_indices_from(w)] = 0.0
    w[np.diag_indices_from(w)] = 1.0 - w.sum(1)
    return w


def laplacian_degrees(graph: nx.Graph) -> np.ndarray:
    """Diagonal of the graph Laplacian as the reference reads it
    (``get_metropolis`` :110-111).  ``nx.laplacian_matrix`` is D - A with D the
    adjacency row sums, so a self loop cancels and L_ii counts proper neighbors."""
    n = graph.number_of_nodes()
    d = np.zeros(n, dtype=np.float64)
    for u, v in graph.edges():
        if u != v:
            d[u] += 1.0
            d[v] += 1.0
    return d


def get_metropolis(graph: nx.Graph, dtype: torch.dtype | None = None) -> torch.Tensor:
    """Metropolis-Hastings mixing matrix of ``graph`` as a ``[N, N]`` tensor
    (reference: utils/graph_generation.py:107-122)."""
    w = metropolis_from_adjacency(adjacency(graph), laplacian_degrees(graph))
    return torch.as_tensor(w, dtype=dtype or torch.get_default_dtype())


def fiedler_value(adj: np.ndarray) -> float:
    """Algebraic connectivity (second smallest Laplacian eigenvalue)."""
    adj = np.asarray(adj, dtype=np.float64)
    if adj.shape[0] < 2:
        return 0.0
    lap = np.diag(adj.sum(1)) - adj
    ev = np.linalg.eigvalsh(lap)
    return float(ev[1])


def is_connected_adj(adj: np.ndarray) -> bool:
    n = adj.shape[0]
    if n == 0:
        return False
    seen = np.zeros(n, dtype=bool)
    frontier = np.zeros(n, dtype=bool)
    frontier[0] = True
    while frontier.any():
        seen |= frontier
        frontier = adj[frontier].any(0) & ~seen
    return bool(seen.all())


def graph_from_adjacency(adj: np.ndarray) -> nx.Graph:
    g = nx.Graph()
    g.add_nodes_from(range(adj.shape[0]))
    iu = np.argwhere(np.triu(adj, 1))
    g.add_edges_from((int(a), int(b)) for a, b in iu)
    return g


# --------------------------------------------------------------------------
# generators (reference API)
# --------------------------------------------------------------------------
def _disk_adjacency(pos: np.ndarray, radius: float) -> np.ndarray:
    d2 = ((pos[:, None, :] - pos[None, :, :]) ** 2).sum(-1)
    adj = d2 <= radius * radius
    np.fill_diagonal(adj, False)
    return adj


def fied_from_disk(N, positions, radius):
    """Fiedler value of the random geometric graph over ``positions`` (a dict
    node -> (x, y) as in the reference :9-11, or an [N,2] array)."""
    pos = _positions_array(N, positions)
    return fiedler_value(_disk_adjacency(pos, radius))


def _positions_array(N, positions) -> np.ndarray:
    if isinstance(positions, dict):
        return np.asarray([positions[i] for i in range(N)], dtype=np.float64)
    return np.asarray(positions, dtype=np.float64).reshape(N, 2)


def _geometric_graph(N, radius, pos: np.ndarray) -> nx.Graph:
    g = graph_from_adjacency(_disk_adjacency(pos, radius))
    nx.set_node_attributes(g, {i: (float(pos[i, 0]), float(pos[i, 1])) for i in range(N)}, "pos")
    return g


def disk_with_fied(N, targ, num_restarts=50, tol=0.01, rng: random.Random | None = None):
    """Random geometric graph on the unit square whose Fiedler value is within
    ``tol`` of ``targ`` — radius bisection as in the reference (:14-66)."""
    rnd = rng or random
    targ = float(targ)
    for _ in range(num_restarts):
        pos = np.asarray([(rnd.random(), rnd.random()) for _ in range(N)], dtype=np.float64)
        lbr, ubr = 0.05, 0.8
        lbf, ubf = fied_from_disk(N, pos, lbr), fied_from_disk(N, pos, ubr)
        if abs(lbf - targ) < tol:
            return _geometric_graph(N, lbr, pos)
        if abs(ubf - targ) < tol:
            return _geometric_graph(N, ubr, pos)
        if not ubf > lbf:
            raise NameError("Degenerate Fiedler bounds in disk graph generation.")
        if targ > ubf or targ < lbf:
            raise NameError("Target outside range.")
        for _c in range(102):
            midr = 0.5 * (ubr + lbr)
            midf = fied_from_disk(N, pos, midr)
            if abs(midf - targ) < tol:
                return _geometric_graph(N, midr, pos)
            if midf > targ:
                ubr = midr
            elif midf < targ:
                lbr = midr
    raise NameError("Never found a viable graph!")


DIRECTED_TYPES = ("directed_cycle", "exponential", "random_directed")


def generate_from_conf(graph_conf) -> Tuple[int, nx.Graph]:
    """Build a graph from a YAML ``graph:`` block (reference :69-104).
    Types: wheel | cycle | complete | random (+ ``p``, ``gen_attempts``), and —
    new here — ``path``, ``star``, ``binary_tree`` (``nx.full_rary_tree(2, N)``:
    node i's children are 2i+1 and 2i+2), ``disk`` (``target_fied``) and the directed
    ``directed_cycle`` (``i -> i+1``), ``exponential`` (``i -> i + 2^m mod N``
    for every ``2^m < N``) and ``random_directed`` (``p``, ``seed``,
    ``gen_attempts``: strongly connected).  Directed graphs (``DIRECTED_TYPES``)
    are an ``nx.DiGraph``; an edge ``u -> v`` means v reads u's row."""
    N = int(graph_conf["num_nodes"])
    kind = graph_conf["type"]
    if kind == "directed_cycle":
        graph = nx.DiGraph()
        graph.add_nodes_from(range(N))
        graph.add_edges_from((i, (i + 1) % N) for i in range(N) if N > 1)
    elif kind == "exponential":
        graph = nx.DiGraph()
        graph.add_nodes_from(range(N))
        m = 1
        while m < N:
            graph.add_edges_from((i, (i + m) % N) for i in range(N))
            m *= 2
    elif kind == "random_directed":
        seed = graph_conf.get("seed", None)
        graph = nx.gnp_random_graph(N, graph_conf["p"], seed=seed, directed=True)
        for k in range(int(graph_conf["gen_attempts"])):
            if nx.is_strongly_connected(graph):
                break
            graph = nx.gnp_random_graph(N, graph_conf["p"], seed=None if seed is None else seed + k + 1, directed=True)
        if not nx.is_strongly_connected(graph):
            raise NameError(
                "A strongly connected random directed graph could not be generated,"
                " increase p or gen_attempts."
            )
    elif kind == "wheel":
        graph = nx.wheel_graph(N)
    elif kind == "cycle":
        graph = nx.cycle_graph(N)
    elif kind == "complete":
        graph = nx.complete_graph(N)
    elif kind == "path":
        graph = nx.path_graph(N)
    elif kind == "star":
        graph = nx.star_graph(N - 1)
    elif kind == "binary_tree":
        graph = nx.full_rary_tree(2, N)
    elif kind == "disk":
        graph = disk_with_fied(N, graph_conf.get("target_fied", 1.0))
    elif kind == "random":
        seed = graph_conf.get("seed", None)
        graph = nx.erdos_renyi_graph(N, graph_conf["p"], seed=seed)
        for k in range(int(graph_conf["gen_attempts"])):
            if nx.is_connected(graph):
                break
            graph = nx.erdos_renyi_graph(
                N, graph_conf["p"], seed=None if seed is None else seed + k + 1
            )
        if not nx.is_connected(graph):
            raise NameError(
                "A connected random graph could not be generated,"
                " increase p or gen_attempts."
            )
    else:
        raise NameError("Unknown communication graph type.")
    return N, graph


def euclidean_disk_graph(poses, radius):
    """Disk graph over ``poses`` [N,2]: edge iff distance <= radius.
    Returns ``(graph, connected)`` (reference :125-146)."""
    pos = np.asarray(poses, dtype=np.float64).reshape(-1, 2)
    adj = _disk_adjacency(pos, float(radius))
    return graph_from_adjacency(adj), is_connected_adj(adj)


def gen_delaunay(N):
    """Graph of the Delaunay triangulation of N uniform points (reference :149)."""
    import scipy.spatial as spatial

    positions = np.random.rand(N, 2)
    tri = spatial.Delaunay(positions)
    edges = set()
    for s in tri.simplices:
        edges.update({(int(s[0]), int(s[1])), (int(s[1]), int(s[2])), (int(s[0]), int(s[2]))})
    return nx.Graph(sorted(edges))


# --------------------------------------------------------------------------
# Topology: cached per-graph tables used by the optimizers / kernels
# --------------------------------------------------------------------------
def topology_key(graph: nx.Graph, adj: np.ndarray | None = None) -> bytes:
    """Identifies the edge set; a directed graph never shares a key with an undirected one."""
    adj = adjacency(graph) if adj is None else adj
    return (b"D" if graph.is_directed() else b"") + adj.tobytes()


class Topology:
    """Immutable view of one communication graph.

    ``neighbors[i]`` follows networkx iteration order (so reference-order
    Gauss-Seidel sweeps visit neighbors exactly as the reference does);
    ``W`` is the float64 Metropolis matrix; ``key`` identifies the edge set so
    callers can cache device tables across rounds (the reference rebuilds W
    every round, SURVEY Q2).

    Every topology also has ``push_weights``, the column-stochastic float64
    matrix ``A_ij = 1 / (d_out(j) + 1)`` of push-sum (SGP), and ``readers[i]``,
    the nodes that read node i's row.  For an undirected graph ``readers`` are
    the neighbors.  For an ``nx.DiGraph`` (``directed``) ``neighbors`` and
    ``neighbors_noself`` are the in-neighbors (the nodes i pulls from),
    ``readers`` the out-neighbors, ``deg`` the in-degrees, and ``W`` is
    ``None``: Metropolis weights are undefined on a directed graph.
    """

    def __init__(self, graph: nx.Graph):
        self.graph = graph
        self.N = graph.number_of_nodes()
        self.directed = graph.is_directed()
        self.adj = adjacency(graph)
        pull = graph.predecessors if self.directed else graph.neighbors
        self.neighbors: List[List[int]] = [
            [int(j) for j in pull(i)] for i in range(self.N)
        ]
        # consensus kernels never treat a node as its own neighbor; the
        # reference would (cycle_graph(1)), which is a no-op for every update.
        self.neighbors_noself = [[j for j in nb if j != i] for i, nb in enumerate(self.neighbors)]
        self.deg = np.asarray([len(nb) for nb in self.neighbors_noself], dtype=np.int64)
        if self.directed:
            self.readers = [[int(j) for j in graph.successors(i) if j != i] for i in range(self.N)]
            self.W = None
        else:
            self.readers = self.neighbors_noself
            self.W = metropolis_from_adjacency(self.adj, laplacian_degrees(graph))
        self.push_weights = push_weights_from_adjacency(self.adj)
        self.key = topology_key(graph, self.adj)

    @property
    def max_degree(self) -> int:
        return int(self.deg.max()) if self.N else 0

    @property
    def max_readers(self) -> int:
        return max((len(r) for r in self.readers), default=0)

    def is_connected(self) -> bool:
        """Connected; strongly connected for a directed graph."""
        return is_strongly_connected_adj(self.adj) if self.directed else is_connected_adj(self.adj)

    def is_complete(self) -> bool:
        return self.N > 1 and bool((self.deg == self.N - 1).all())

    def reverse_slots(self) -> List[List[int]]:
        """``rs[i][e]``: the position of i in ``neighbors_noself[j]`` for ``j = neighbors_noself[i][e]`` (undirected
        graphs), the slot under which neighbor j keeps what it exchanges with i."""
        pos = [{j: e for e, j in enumerate(nb)} for nb in self.neighbors_noself]
        return [[pos[j][i] for j in nb] for i, nb in enumerate(self.neighbors_noself)]

    def reach_table(self) -> np.ndarray:
        """``R[i, k] = |{l : d(i, l) <= k}|`` (i itself included) for ``k = 0 .. diam``, by breadth-first search from
        every node; ``diam`` is the largest finite hop distance, so ``R[:, -1]`` is each node's component size."""
        dist = np.full((self.N, self.N), -1, dtype=np.int64)
        for s in range(self.N):
            dist[s, s] = 0
            frontier = [s]
            while frontier:
                nxt = []
                for u in frontier:
                    for v in self.neighbors_noself[u]:
                        if dist[s, v] < 0:
                            dist[s, v] = dist[s, u] + 1
                            nxt.append(v)
                frontier = nxt
        diam = int(dist.max()) if self.N else 0
        return np.stack([((dist >= 0) & (dist <= k)).sum(1) for k in range(diam + 1)], axis=1)

    def is_tree(self) -> bool:
        """Undirected, connected and exactly ``N - 1`` edges."""
        return not self.directed and self.is_connected() and int(self.adj.sum()) // 2 == self.N - 1

    def padded_table(self, dmax: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """(nbr_idx [N,dmax] int32 (-1 pad), nbr_w [N,dmax] f64, self_w [N] f64, deg [N] int32)."""
        idx = -np.ones((self.N, dmax), dtype=np.int32)
        w = np.zeros((self.N, dmax), dtype=np.float64)
        for i, nb in enumerate(self.neighbors_noself):
            idx[i, : len(nb)] = nb
            w[i, : len(nb)] = self.W[i, nb]
        return idx, w, np.diag(self.W).copy(), self.deg.astype(np.int32)


class TopologyCache:
    """Maps graphs to ``Topology`` objects, keyed by edge set."""

    def __init__(self):
        self._by_key: Dict[bytes, Topology] = {}

    def get(self, graph: nx.Graph) -> Topology:
        key = topology_key(graph)
        topo = self._by_key.get(key)
        if topo is None:
            topo = Topology(graph)
            self._by_key[key] = topo
        return topo
