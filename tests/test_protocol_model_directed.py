"""Model check of the publication protocol on directed graphs (ops/csrc/consensus_device.cuh: begin_round /
wait_neighbors with reader tables), with the explorer of tests/test_protocol_model.py — CPU only, no kernels: every
rank is a small state machine and all interleavings of a few rounds are explored.

Protocol of rank r in round k (published rows double buffered by round parity), on a directed graph where r pulls from
its in-neighbors in_k(r) and its row is read by its out-neighbors out_k(r):
  announce   flag[r] = k                      (its row of round k was written at the end of round k-1)
  wait       until flag[j] >= k for every j in in_k(r)  [+ out_{k-1}(r): the rank that read the buffer r overwrites]
  read       pub[j][k & 1] for every j in in_k(r), one at a time
  write      pub[r][(k+1) & 1] = row of round k+1
Safety: every read returns the row of round k; liveness: no deadlock."""
import itertools
import random

from test_protocol_model import directed_waits, explore_sets


def explore(ins, n_ranks, wait_readers, announce_at_start=True, max_states=400_000):
    """The directed protocol: ins[k][r] = in-neighbor ranks of r in round k; r waits for in_k(r), and with
    ``wait_readers`` also for out_{k-1}(r)."""
    return explore_sets(ins, directed_waits(ins, n_ranks, wait_readers), n_ranks, announce_at_start, max_states)


def _ring(n):
    """Directed ring r -> r + 1: rank r pulls from r - 1 and is read by r + 1."""
    return [{(r - 1) % n} for r in range(n)]


def _union_with_undirected(ins):
    return [set(s) | {j for j in range(len(ins)) if r in ins[j]} for r, s in enumerate(ins)]


def test_waiting_only_on_in_neighbors_is_unsafe_on_a_static_directed_ring():
    """A rank waits for nobody downstream, runs ahead of its reader and overwrites the buffer still being read."""
    for n in (3, 4):
        v, d, _ = explore([_ring(n)] * (n + 1), n, wait_readers=False, max_states=300_000)
        assert d is None
        assert v is not None, n
        r, k, j, tag = v
        assert tag == k + 2, v          # rows written two rounds ahead in the buffer the reader still uses


def test_in_and_readers_wait_is_safe_on_static_directed_graphs():
    for n in (3, 4):
        for at_start in (True, False):
            v, d, states = explore([_ring(n)] * 3, n, wait_readers=True, announce_at_start=at_start, max_states=300_000)
            assert v is None and d is None, (n, at_start, v, d)
            assert 100 < states < 300_000     # branched, and exhaustive (not cut off)
    expo = [{(r - 1) % 4, (r - 2) % 4} for r in range(4)]       # exponential graph of 4 ranks: in-degree 2
    v, d, states = explore([expo] * 3, 4, wait_readers=True, max_states=300_000)
    assert v is None and d is None and states < 300_000


def test_on_undirected_graphs_the_set_is_the_union_wait():
    """For a symmetric graph out_{k-1} = N_{k-1}: the wait is the undirected protocol's N_k and N_{k-1}."""
    sym = _union_with_undirected(_ring(4))
    v, d, states = explore([sym] * 3, 4, wait_readers=True, max_states=300_000)
    assert v is None and d is None and states < 300_000


MAX_RANDOM = 200_000


def test_random_time_varying_digraphs_random_schedules():
    """Random digraphs per round (ranks without in-neighbors included), both announcement points."""
    rng = random.Random(5)
    for trial in range(40):
        n = rng.choice([3, 4])
        K = 3
        pairs = [(a, b) for a, b in itertools.permutations(range(n), 2)]
        graphs = []
        for _ in range(K):
            ins = [set() for _ in range(n)]
            for a, b in pairs:
                if rng.random() < 0.4:
                    ins[b].add(a)
            graphs.append(ins)
        v, d, states = explore(graphs, n, wait_readers=True, announce_at_start=bool(trial & 1), max_states=MAX_RANDOM)
        assert v is None and d is None, (trial, graphs, v, d)
        assert states < MAX_RANDOM, (trial, graphs)      # the search finished: safe in every interleaving
