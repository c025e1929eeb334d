"""Model check of the cross-GPU publication protocol (ops/csrc/consensus_device.cuh: begin_round / wait_neighbors /
finish_round) — CPU only, no kernels: every rank is a small state machine and ALL interleavings of a few rounds on a
time-varying graph are explored.  This file holds the explorer and the undirected cases;
tests/test_protocol_model_directed.py runs the same explorer on directed graphs.

Protocol of rank r in round k (published rows are double buffered by round parity):
  announce   flag[r] = k                      (its rows of round k were written at the end of round k-1)
  wait       until flag[j] >= k for every j in N_k(r)  [+ N_{k-1}(r): the write-after-read fix]
  read       pub[j][k & 1] for every j in N_k(r), one neighbor at a time
  write      pub[r][(k+1) & 1] = rows of round k+1
On a directed graph the reads are from in_k(r) and the fix waits for out_{k-1}(r), the readers of the buffer being
overwritten; N_k and N_{k-1} are what those sets are on an undirected graph, and wait_neighbors is one function.
Safety: every read returns the rows of round k (never rows of k+2 written early, never stale ones); liveness: no deadlock.
The reference has no counterpart (one process, optimizers/dinno.py:103-110 snapshots all replicas at once); the
hazard only exists because ranks run free of each other between flag waits."""
import itertools
import random

import pytest

from nn_distributed_training_b200.ops.engine import WAIT_THREADS, check_wait_capacity


def explore_sets(reads, waits, n_ranks, announce_at_start=True, max_states=400_000):
    """DFS over all interleavings of the protocol with explicit sets: rank r reads ``reads[k][r]`` in round k after
    waiting for "round k published" from ``waits[k][r]``.  Returns (violation, deadlock, n_states)."""
    K = len(reads)

    def program(r):                                                # list of atomic steps
        steps = []
        for k in range(K):
            if announce_at_start:
                steps.append(("announce", k))
            steps.append(("wait", k, tuple(sorted(waits[k][r]))))
            for j in sorted(reads[k][r]):
                steps.append(("read", k, j))
            steps.append(("write", k))
            if not announce_at_start:
                steps.append(("announce", k + 1))
        return steps

    progs = [program(r) for r in range(n_ranks)]
    init = (tuple(0 for _ in range(n_ranks)),                      # pc per rank
            tuple(0 for _ in range(n_ranks)),                      # flag per rank
            tuple((0, -1) for _ in range(n_ranks)))                # pub[r] = (tag of parity 0, tag of parity 1)
    seen = {init}
    stack = [init]
    while stack and len(seen) < max_states:
        pcs, flags, pubs = stack.pop()
        progressed = False
        done = True
        for r in range(n_ranks):
            if pcs[r] >= len(progs[r]):
                continue
            done = False
            st = progs[r][pcs[r]]
            nflags, npubs = flags, pubs
            if st[0] == "announce":
                nflags = flags[:r] + (max(flags[r], st[1]),) + flags[r + 1:]
            elif st[0] == "wait":
                if any(flags[j] < st[1] for j in st[2]):
                    continue                                        # blocked
            elif st[0] == "read":
                k, j = st[1], st[2]
                if pubs[j][k & 1] != k:
                    return (r, k, j, pubs[j][k & 1]), None, len(seen)
            elif st[0] == "write":
                k = st[1]
                p = list(pubs[r]); p[(k + 1) & 1] = k + 1
                npubs = pubs[:r] + (tuple(p),) + pubs[r + 1:]
            progressed = True
            nxt = (pcs[:r] + (pcs[r] + 1,) + pcs[r + 1:], nflags, npubs)
            if nxt not in seen:
                seen.add(nxt)
                stack.append(nxt)
        if not done and not progressed:
            return None, (pcs, flags), len(seen)
    return None, None, len(seen)


def undirected_waits(graphs, n_ranks, wait_prev=True):
    """wait_neighbors without reader tables: N_k(r), and with ``wait_prev`` also N_{k-1}(r)."""
    return [[set(graphs[k][r]) | (set(graphs[k - 1][r]) if (wait_prev and k > 0) else set()) for r in range(n_ranks)]
            for k in range(len(graphs))]


def directed_waits(ins, n_ranks, wait_readers=True):
    """wait_neighbors with reader tables: in_k(r), and with ``wait_readers`` also out_{k-1}(r), the ranks that read
    the buffer r overwrites at the end of round k."""
    outs = [[{j for j in range(n_ranks) if r in g[j]} for r in range(n_ranks)] for g in ins]
    return [[set(ins[k][r]) | (outs[k - 1][r] if (wait_readers and k > 0) else set()) for r in range(n_ranks)]
            for k in range(len(ins))]


def explore(graphs, n_ranks, wait_prev, announce_at_start=True, max_states=400_000):
    """The undirected protocol: graphs[k][r] = set of neighbor ranks of r in round k."""
    return explore_sets(graphs, undirected_waits(graphs, n_ranks, wait_prev), n_ranks, announce_at_start, max_states)


def _sym(n, edges):
    g = [set() for _ in range(n)]
    for a, b in edges:
        g[a].add(b); g[b].add(a)
    return g


# rank 1 is a neighbor of rank 0 in round 0 only: the case VERDICT weak #4 describes
DYNAMIC = [_sym(3, [(0, 1), (0, 2)]), _sym(3, [(0, 2)]), _sym(3, [(0, 2), (1, 2)]), _sym(3, [(0, 1)])]


def test_waiting_only_on_current_neighbors_is_unsafe_on_time_varying_graphs():
    v, d, n = explore(DYNAMIC, 3, wait_prev=False)
    assert d is None
    assert v is not None, "the model must reproduce the write-after-read hazard of the round-1 protocol"
    r, k, j, tag = v
    assert tag == k + 2          # the reader found rows written two rounds ahead in the buffer it was still reading


def test_union_wait_closes_the_window_for_both_announcement_points():
    for at_start in (True, False):
        v, d, n = explore(DYNAMIC, 3, wait_prev=True, announce_at_start=at_start)
        assert v is None and d is None, (at_start, v, d)
        assert 300 < n < 400_000     # the search branched and was exhaustive (not cut off by max_states)


def test_static_graphs_need_no_extra_wait():
    ring = [_sym(4, [(0, 1), (1, 2), (2, 3), (3, 0)])] * 3
    for wait_prev in (False, True):
        v, d, n = explore(ring, 4, wait_prev=wait_prev, max_states=300_000)
        assert v is None and d is None and n < 300_000


def test_random_time_varying_graphs_random_schedules():
    """Larger instances than the exhaustive search can cover: random graphs per round, the union wait, both announcement
    points; isolated ranks (no neighbors in a round) included."""
    rng = random.Random(3)
    for trial in range(40):
        n = rng.choice([3, 4, 5])
        K = 3
        pairs = list(itertools.combinations(range(n), 2))
        graphs = [_sym(n, [e for e in pairs if rng.random() < 0.5]) for _ in range(K)]
        v, d, _ = explore(graphs, n, wait_prev=True, announce_at_start=bool(trial & 1), max_states=60_000)
        assert v is None and d is None, (trial, graphs, v, d)


def test_the_directed_rule_gives_the_undirected_wait_sets_on_undirected_graphs():
    """With in = out = N the sets in_k + out_{k-1} are N_k + N_{k-1}: wait_neighbors without reader tables (neighbor
    tables of graph_id[k-1]) waits for exactly what it would with the neighbor tables passed as reader tables."""
    rng = random.Random(7)
    for trial in range(200):
        n = rng.choice([2, 3, 4, 5, 6])
        pairs = list(itertools.combinations(range(n), 2))
        graphs = [_sym(n, [e for e in pairs if rng.random() < 0.5]) for _ in range(4)]
        if trial & 1:
            graphs[2] = graphs[1]                                   # a repeated graph: the set step 1 already waited for
        for fix in (True, False):
            assert directed_waits(graphs, n, fix) == undirected_waits(graphs, n, fix), (trial, graphs)


def test_a_node_with_more_peers_than_waiting_threads_is_rejected():
    """The wait has one thread per in-neighbor (from thread 0) and one per reader (from thread 32) of a CTA."""
    check_wait_capacity(1, 0)
    check_wait_capacity(WAIT_THREADS, WAIT_THREADS - 32)
    with pytest.raises(ValueError, match="in-neighbors"):
        check_wait_capacity(WAIT_THREADS + 1, 1)
    with pytest.raises(ValueError, match="readers"):
        check_wait_capacity(3, WAIT_THREADS - 31)
