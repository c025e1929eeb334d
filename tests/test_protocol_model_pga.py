"""Model check of Gossip-PGA's publication protocol (ops/csrc/consensus.cu: pga_sum_kernel / pga_mix_kernel,
consensus_device.cuh: pga_phase) — CPU only, no kernels.  The explorer of tests/test_protocol_model.py, extended with
the fp64 partial-sum buffers of the global rounds: every rank is a small state machine and the interleavings of a few
rounds are explored depth first.

Rank r in round k (published rows double buffered by round parity, partial sums by `sum_par(k)`):
  gossip round  announce flag[r] = k; wait flag[j] >= k for j in N_k(r) + N_{k-1}(r); read pub[j][k & 1] for j in N_k(r)
                (none with gossip: false, the edgeless graph); write pub[r][(k+1) & 1]
  global round  write part[r][sum_par(k)]; post sumflag[r] = k + 1; announce flag[r] = k;
                wait sumflag[j] >= k + 1 for every j; read part[j][sum_par(k)] for every j; write pub[r][(k+1) & 1]
Safety: every read of a published row returns round k's and every read of a partial sum returns global round k's;
liveness: no deadlock.  Indexing the partials by round parity (k & 1) is unsafe once global rounds are `period` apart;
indexing them by the global round's count (k / period) & 1 is what the kernels do."""
import itertools
import random

from test_protocol_model import _sym, undirected_waits


def explore_pga(graphs, n_ranks, period, gossip=True, count_parity=True, max_states=400_000):
    """DFS over the interleavings of ``len(graphs)`` rounds; ``graphs[k][r]`` is the base-graph neighbor set of rank r in
    round k (ignored on global rounds and with ``gossip`` false).  Returns (violation, deadlock, n_states)."""
    K = len(graphs)
    glob = [k % period == period - 1 for k in range(K)]
    nbrs = graphs if gossip else [[set() for _ in range(n_ranks)] for _ in range(K)]
    waits = undirected_waits(nbrs, n_ranks)

    def sum_par(k):
        return (k // period) & 1 if count_parity else k & 1

    def program(r):
        steps = []
        for k in range(K):
            if glob[k]:
                steps += [("part", k), ("post", k), ("announce", k), ("swait", k)]
                steps += [("sread", k, j) for j in range(n_ranks)]
            else:
                steps += [("announce", k), ("wait", k, tuple(sorted(waits[k][r])))]
                steps += [("read", k, j) for j in sorted(nbrs[k][r])]
            steps.append(("write", k))
        return steps

    progs = [program(r) for r in range(n_ranks)]
    z = tuple(0 for _ in range(n_ranks))
    init = (z, z, z,                                                # pc, flag, sum flag per rank
            tuple((0, -1) for _ in range(n_ranks)),                 # pub[r] = round tag of parity 0, 1
            tuple((-1, -1) for _ in range(n_ranks)))                # part[r] = round tag of buffer 0, 1
    seen = {init}
    stack = [init]
    while stack and len(seen) < max_states:
        pcs, flags, sflags, pubs, parts = stack.pop()
        progressed, done = False, True
        for r in range(n_ranks):
            if pcs[r] >= len(progs[r]):
                continue
            done = False
            st = progs[r][pcs[r]]
            k = st[1]
            nf, ns, npub, npart = flags, sflags, pubs, parts
            if st[0] == "announce":
                nf = flags[:r] + (max(flags[r], k),) + flags[r + 1:]
            elif st[0] == "wait":
                if any(flags[j] < k for j in st[2]):
                    continue
            elif st[0] == "read":
                if pubs[st[2]][k & 1] != k:
                    return ("pub", r, k, st[2], pubs[st[2]][k & 1]), None, len(seen)
            elif st[0] == "part":
                p = list(parts[r]); p[sum_par(k)] = k
                npart = parts[:r] + (tuple(p),) + parts[r + 1:]
            elif st[0] == "post":
                ns = sflags[:r] + (k + 1,) + sflags[r + 1:]
            elif st[0] == "swait":
                if any(sflags[j] < k + 1 for j in range(n_ranks) if j != r):
                    continue
            elif st[0] == "sread":
                if parts[st[2]][sum_par(k)] != k:
                    return ("sum", r, k, st[2], parts[st[2]][sum_par(k)]), None, len(seen)
            elif st[0] == "write":
                p = list(pubs[r]); p[(k + 1) & 1] = k + 1
                npub = pubs[:r] + (tuple(p),) + pubs[r + 1:]
            progressed = True
            nxt = (pcs[:r] + (pcs[r] + 1,) + pcs[r + 1:], nf, ns, npub, npart)
            if nxt not in seen:
                seen.add(nxt)
                stack.append(nxt)
        if not done and not progressed:
            return None, (pcs, flags, sflags), len(seen)
    return None, None, len(seen)


PATH3 = _sym(3, [(0, 1), (1, 2)])


def test_round_parity_partials_are_overwritten_before_a_far_rank_reduces_them():
    """Period 2 on a 3-rank path: every global round (k = 1, 3, 5) lands on the same round parity.  Rank 0 finishes
    global round 1, gossips with rank 1 in round 2 and overwrites its partial in global round 3 while rank 2, two hops
    away, still reduces global round 1."""
    v, d, _ = explore_pga([PATH3] * 4, 3, period=2, count_parity=False)
    assert d is None
    assert v is not None and v[0] == "sum", v
    _, r, k, j, tag = v
    assert k == 1 and tag == 3        # a partial of global round 3 read in place of round 1's


def test_global_count_parity_is_safe_on_paths_and_cycles():
    for n in (3, 4):
        path = _sym(n, [(i, i + 1) for i in range(n - 1)])
        cycle = _sym(n, [(i, (i + 1) % n) for i in range(n)])
        for period in (1, 2, 3, 4):
            K = 2 * period + 1 if n == 3 else period + 2      # at least two global rounds (three on 3 ranks)
            for graph in (path, cycle):
                for gossip in (True, False):
                    v, d, states = explore_pga([graph] * K, n, period, gossip=gossip, max_states=400_000)
                    assert v is None and d is None, (n, period, gossip, v, d)
                    assert states < 400_000, (n, period, gossip)     # exhaustive, not cut off


def test_global_count_parity_on_random_time_varying_graphs():
    """Random base graphs per round (isolated ranks included), periods 1 to 4; larger than an exhaustive search covers,
    so the search is bounded."""
    rng = random.Random(11)
    for trial in range(40):
        n = rng.choice([3, 4])
        period = rng.choice([1, 2, 3, 4])
        K = period + 3
        pairs = list(itertools.combinations(range(n), 2))
        graphs = [_sym(n, [e for e in pairs if rng.random() < 0.5]) for _ in range(K)]
        v, d, _ = explore_pga(graphs, n, period, gossip=bool(trial & 1), max_states=60_000)
        assert v is None and d is None, (trial, period, graphs, v, d)
