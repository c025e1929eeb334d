"""RelaySum on the fused sm_90a kernels: ``relay_mix_kernel`` and ``relay_step_kernel`` one launch at a time against a
float64 oracle of the definition with the bound of ``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err), then
CUDA-graph replay, whole runs against the PyTorch path, the input pipelines, determinism, checkpoint/resume, the sequence
check and the refusal of a changing graph."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import relaysum_oracle as ro
from test_gpu_consensus_kernels import S_LIST, VEC, KernelProblem, _snap
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import RelaySum
from nn_distributed_training_b200.utils.graph_generation import Topology, generate_from_conf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


def _gen(kind, N):
    return generate_from_conf({"type": kind, "num_nodes": N})[1]


def _permuted_tree():
    """A binary tree of 10 nodes under a random relabelling, its edges inserted in random order: neighbor lists in no
    particular order, so a wrong reverse slot reads another neighbor's message."""
    rng = np.random.default_rng(5)
    perm = rng.permutation(10)
    edges = [(int(perm[a]), int(perm[b])) for a, b in _gen("binary_tree", 10).edges()]
    rng.shuffle(edges)
    g = nx.Graph()
    g.add_nodes_from(range(10))
    g.add_edges_from(edges)
    return g


def _prufer_tree():
    rng = np.random.default_rng(11)
    return nx.from_prufer_sequence([int(x) for x in rng.integers(0, 9, size=7)])


# degrees 0 (one node), 1 (every leaf, path2: the complete K2 on the pointer table), 2, 3 and the star hubs 4 .. 9
TREES = {
    "single": nx.empty_graph(1), "path2": _gen("path", 2), "path10": _gen("path", 10),
    "binary_tree10": _gen("binary_tree", 10), "permuted": _permuted_tree(), "prufer9": _prufer_tree(),
    "star5": _gen("star", 5), "star10": _gen("star", 10),
}
ROUNDS = 11          # past ecc(i) of every node (path10: 9)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:28s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(key, dtype, S, n, n_pad=None, seed=0, rounds=ROUNDS):
    conf = {"alg_name": "relaysum", "alpha0": 0.05, "mu": 0.5, "outer_iterations": rounds, "profile": False}
    pr = KernelProblem([TREES[key]], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, RelaySum(pr, DEV, conf), conf


def _state(pr, o, eng):
    s = _snap(pr, o, eng)
    s["rin"] = eng.rin.detach().double().cpu().numpy().copy()
    return s


class Harness:
    def __init__(self, pr, o):
        self.pr, self.o = pr, o
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        t = Topology(pr.graph)
        self.nbrs, self.rs = t.neighbors_noself, t.reverse_slots()
        self.R = t.reach_table()
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.alpha = self.eng.alpha.cpu().double().numpy()
        assert not self.eng.sum_mode and self.eng.C == max(1, t.max_degree)
        self.n = pr.n

    def mix(self, st, k):
        par, u, N = k & 1, self.u, self.pr.N
        out = dict(st, theta=st["theta"].copy(), rin=st["rin"].copy())
        err = {"theta": np.zeros_like(st["theta"]), "rin": np.zeros_like(st["rin"])}
        for i in range(N):
            h = st["theta"][i]
            r = [st["pub"][par, self.rs[i][e], j] for e, j in enumerate(self.nbrs[i])]
            s, mag = np.zeros_like(h), np.zeros_like(h)
            for e, q in enumerate(r):
                s = s + q
                mag = mag + np.abs(q)
                out["rin"][i, e] = q
            c = float(self.R[i, min(k, self.R.shape[1] - 1)] - 1)
            q = (s - c * h) / N
            out["theta"][i] = h + q
            e_s = u * len(r) * mag
            err["theta"][i] = (e_s + u * (np.abs(c * h) + np.abs(s - c * h))) / N + u * (np.abs(q) + np.abs(h + q))
        return out, err

    def step(self, st, k):
        par, u = k & 1, self.u
        a = self.alpha[k]
        g, e_g = co.sum_partials(st["grad_part"], u)
        h = st["theta"] - a * g
        e_h = a * e_g + u * (np.abs(st["theta"]) + 2.0 * a * np.abs(g))
        pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
        for i, nb in enumerate(self.nbrs):
            r = st["rin"][i, :len(nb)]
            for e in range(len(nb)):
                m, mag = h[i].copy(), np.abs(h[i])
                for f in range(len(nb)):
                    if f != e:
                        m = m + r[f]
                        mag = mag + np.abs(r[f])
                pub[par ^ 1, e, i] = m
                e_pub[par ^ 1, e, i] = e_h[i] + u * len(nb) * mag
        return dict(st, theta=h, pub=pub), {"theta": e_h, "pub": e_pub}

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        step = name == "relay_step"
        assert after["done_ctr"] == 0, name
        assert after["round_ctr"] == before["round_ctr"] + (1 if step else 0), name
        assert not after["theta"][..., self.n:].any(), f"{name}: padding of theta written"
        if not check:
            return
        want, err = self.step(before, k) if step else self.mix(before, k)
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name} round {k} {key}", got, want[key], err[key], C)
                WORST[(name, self.dt)] = max(WORST[(name, self.dt)], r)
            else:
                assert np.array_equal(got, before[key]), f"{name} round {k} wrote {key}"

    def run(self, rounds=ROUNDS, checked=None):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = checked is None or k in checked
            self.launch("relay_mix", op.relay_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("relay_step", op.relay_step, k, check=chk)
        self.eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("key", sorted(TREES))
def test_launches_match_oracle(key, dtype):
    """Every tree (degrees 0 .. 9, a relabelled tree whose neighbor lists are in no order), rounds before and after
    every node's eccentricity, with garbage in rin before the first mix and S rotating with the case."""
    i = sorted(TREES).index(key)
    pr, o, _ = _setup(key, dtype, S_LIST[i % len(S_LIST)], 13, seed=i)
    h = Harness(pr, o)
    h.eng.rin.copy_(torch.randn(h.eng.rin.shape, dtype=torch.float64).to(dtype) * 1e3)
    h.run()


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The 4-deep and 8-deep partial sums on a binary tree, the 4-deep one with the tail loop on the star hub."""
    for key in ("binary_tree10", "star10"):
        pr, o, _ = _setup(key, dtype, S, 77, seed=S, rounds=4)
        Harness(pr, o).run(rounds=4)


@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, _ = _setup("star10", dtype, 5, vec, n_pad=vec, seed=3)
        Harness(pr, o).run()
        return
    if size == "padded":
        pr, o, _ = _setup("permuted", dtype, 3, 9, n_pad=64 * vec, seed=5)
        Harness(pr, o).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, _ = _setup("binary_tree10", dtype, 17, 140001, seed=4, rounds=3)
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o).run(rounds=3)


@pytest.mark.parametrize("key", ["binary_tree10", "star10"])
def test_graph_replay_equals_eager_launches(key):
    runs = []
    for capture in (False, True):
        pr, o, _ = _setup(key, torch.float32, 5, 300, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        assert prog.launches_per_round() == 3 and prog.dpr == 1
        assert prog.pr._metric_engine is None
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            states.append(_state(pr, o, prog.eng))
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key_, x in a.items():
            if isinstance(x, np.ndarray):
                assert np.array_equal(x, b[key_]), f"round {k}: {key_}"
            else:
                assert x == b[key_], f"round {k}: {key_}"


def test_bytes_per_round_are_dsgd_s():
    pr, o, _ = _setup("binary_tree10", torch.float64, 1, 100)
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    row = pr.arena.n_pad * 8
    assert eng.bytes_per_round() == {"row": row, "pulled": row * 2 * 9}


def test_a_multi_topology_plan_is_refused():
    pr, o, _ = _setup("path10", torch.float32, 1, 20)
    with pytest.raises(ValueError, match="relaysum needs a fixed tree"):
        ConsensusEngine(o, [nx.path_graph(10), _gen("binary_tree", 10)] * 3)


# ------------------------------------------------------------------------------------------ whole runs ----
RS = {"alg_name": "relaysum", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _tree(monkeypatch, kind, N):
    """The test problems build ``nx.cycle_graph(N)``: hand them a tree instead."""
    monkeypatch.setattr(nx, "cycle_graph", lambda n: _gen(kind, n))


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    return RelaySum(a, DEV, copy.deepcopy(conf)), RelaySum(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))


@pytest.mark.parametrize("kind", ["path", "binary_tree"])
def test_mnist_fp64_paper_shape_matches_torch_fp64(monkeypatch, kind):
    from test_gpu_mnist import _generic_problem
    _tree(monkeypatch, kind, 6)
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=6, eval_every=3, conf=copy.deepcopy(RS))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=6, eval_every=3, conf=copy.deepcopy(RS))
    oa, ob = _pair(a, b, RS)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    oa._program.sync_back()
    rm = _rel(oa.msg, ob.msg)
    print(f"\nMNIST fp64 relaysum on {kind}: rel theta {r:.2e}, msg {rm:.2e}")
    assert r < 1e-8 and rm < 1e-8
    assert a.forward_cnt == b.forward_cnt


def test_density_fp64_matches_torch_fp64(monkeypatch):
    from test_gpu_mlp_f64 import _density
    _tree(monkeypatch, "binary_tree", 4)
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(RS))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(RS))
    oa, ob = _pair(a, b, RS)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64 relaysum: rel {r:.2e}")
    assert r < 1e-8
    oa._program.sync_back()
    assert _rel(oa.msg, ob.msg) < 1e-8
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(RS, outer_iterations=12)
        pr = _problem(5, 32, "fused", conf, M=100, eval_every=1000, graph=_gen("binary_tree", 5))
        pr.conf["input_pipeline"] = pl
        opt = RelaySum(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.msg.clone(), pr.forward_cnt, pr.calls.copy()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][2] == outs[1][2] and (outs[0][3] == outs[1][3]).all()


def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", dict(RS), graph=_gen("star", 5), eval_every=3)
        opt = RelaySum(pr, DEV, dict(RS))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.msg.clone()))
    for run in outs[1:]:
        assert torch.equal(run[0], outs[0][0]) and torch.equal(run[1], outs[0][1])


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, monkeypatch, model):
    """Resume at round 3: the published messages come back from the checkpoint into the other parity's buffer."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(RS, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(5, 32, "fused", conf, M=100, graph=_gen("binary_tree", 5))
    else:
        from test_gpu_mlp_f64 import _density
        _tree(monkeypatch, "path", 4)

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = RelaySum(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = RelaySum(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3 and o1.msg.any()
    second = make()
    o2 = RelaySum(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.msg, of.msg)
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes():
    """``debug_sequence_check``: every message read is tagged with the round it belongs to, and the run matches the
    PyTorch ops."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        pr = _problem(6, 32, "fused", dict(RS), graph=_gen("binary_tree", 6), eval_every=1000)
        c = dict(RS, debug_sequence_check=True, consensus_backend="auto" if backend == "fused" else "torch")
        opt = RelaySum(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert opt._program.eng.seq_buf is not None
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
