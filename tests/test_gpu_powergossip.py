"""PowerGossip on the fused sm_90a kernels: ``pg_mix_kernel`` and ``pg_step_kernel`` one launch at a time against the
float64 oracle of ``tests/powergossip_oracle.py`` (|kernel - oracle| <= 16 u err) for degrees 1 .. 16 in both phases,
the endpoint vectors bit-equal after every mix, messages that do not depend on the grid, CUDA-graph replay, whole runs
against the PyTorch path, determinism, the input pipelines, checkpoint/resume, the sequence check and the capacity
refusal."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import powergossip_oracle as po
from test_gpu_consensus_kernels import KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine, check_powergossip_capacity
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import PowerGossip
from nn_distributed_training_b200.parallel.arena import FlatLayout, ParamSlot
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


def _random():
    for seed in range(1000):
        g = nx.gnp_random_graph(9, 0.4, seed=seed)
        if nx.is_connected(g):
            return g
    raise AssertionError


# largest degree 1 (path2), 2 (cycle6), 4 (complete5), 8 (wheel9 hub), 16 (star17 hub), a random graph
GRAPHS = {"path2": nx.path_graph(2), "cycle6": nx.cycle_graph(6), "complete5": nx.complete_graph(5),
          "wheel9": nx.wheel_graph(9), "star17": nx.star_graph(16), "random9": _random()}
SMALL = [(6, 5), (6,), (3, 2, 4), (3,)]
LARGE = [(40, 150), (40,), (7, 3, 30), (7,)]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:10s} {dt:5s} {r:.3f}")


class PgProblem(KernelProblem):
    """KernelProblem with a row of matrices and biases (dense slots, so no holes)."""

    def __init__(self, graph, dtype, S, seed, shapes, conf):
        slots, off = [], 0
        for k, sh in enumerate(shapes):
            numel = int(np.prod(sh))
            slots.append(ParamSlot(f"p{k}", tuple(sh), off, numel))
            off += numel
        super().__init__([graph], off, dtype, S, seed=seed, conf=conf)
        lay = FlatLayout(slots)
        assert lay.n_pad == self.layout.n_pad
        self.layout = self.arena.layout = lay


def _setup(key, dtype, S=3, seed=0, shapes=SMALL, rounds=6, **kw):
    conf = dict({"alg_name": "powergossip", "alpha0": 0.05, "mu": 0.5, "gamma": 0.8, "outer_iterations": rounds,
                 "profile": False}, **kw)
    pr = PgProblem(GRAPHS[key], dtype, S, seed, shapes, conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :pr.n] = torch.randn(pr.N, pr.n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, PowerGossip(pr, DEV, conf), conf


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def _endpoints_equal(o, nbrs, rs):
    vec = o.vec.cpu()
    for i, nb in enumerate(nbrs):
        for e, j in enumerate(nb):
            assert torch.equal(vec[i, e], vec[j, rs[i][e]]), f"vectors of edge ({i}, {j}) differ between its endpoints"


class Harness:
    def __init__(self, pr, o):
        self.pr, self.o = pr, o
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        t = Topology(pr.graph)
        self.nbrs, self.rs, self.W = t.neighbors_noself, t.reverse_slots(), t.W
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.alpha = self.eng.alpha.cpu().double().numpy()
        self.lay = o.lay
        assert not self.eng.sum_mode and self.eng.C == max(1, t.max_degree)

    def state(self):
        return dict(theta=_t(self.pr.arena.theta), vec=_t(self.o.vec), pub=_t(self.eng.pub[:, :, :self.pr.N]),
                    grad_part=_t(self.pr.fused.grad_part))

    def _check(self, name, k, got, want, err):
        r = co.check(f"{name} round {k}", got, want, err, C)
        WORST[(name, self.dt)] = max(WORST[(name, self.dt)], r)

    def run(self, rounds):
        op, lay = self.eng.op, self.lay
        for k in range(rounds):
            par = k & 1
            st = self.state()
            op.pg_mix()
            torch.cuda.synchronize()
            got = self.state()
            pub = st["pub"][par].transpose(1, 0, 2)                  # [N, dmax, W]
            x, ex, vn, ev = po.mix(st["theta"], st["vec"], pub, self.nbrs, self.rs, self.W, self.o.gamma, lay.segs,
                                   lay.P, lay.Q, par, self.u)
            self._check("pg_mix", k, got["theta"], x, ex)
            self._check("pg_mix", k, got["vec"], vn, ev)
            assert np.array_equal(got["pub"], st["pub"]), f"pg_mix round {k} wrote the published buffer"
            _endpoints_equal(self.o, self.nbrs, self.rs)
            self.pr.fused.launch()
            st = self.state()
            op.pg_step()
            torch.cuda.synchronize()
            got = self.state()
            g, e_g = co.sum_partials(st["grad_part"], self.u)
            nxt = st["pub"][par ^ 1].transpose(1, 0, 2)
            h, eh, msg, em = po.step(st["theta"], g, e_g, self.alpha[k], st["vec"], nxt, self.nbrs, lay.segs, lay.P,
                                     lay.Q, par ^ 1, self.u)
            self._check("pg_step", k, got["theta"], h, eh)
            self._check("pg_step", k, got["pub"][par ^ 1].transpose(1, 0, 2), msg, em)
            assert np.array_equal(got["pub"][par], st["pub"][par]), f"pg_step round {k} wrote the round's parity"
            assert int(self.eng.round_ctr.item()) == k + 1 and int(self.eng.done_ctr.item()) == 0
        self.eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("key", sorted(GRAPHS))
def test_launches_match_oracle(key, dtype):
    i = sorted(GRAPHS).index(key)
    pr, o, _ = _setup(key, dtype, S=1 + i % 5, seed=i)
    Harness(pr, o).run(4)


@DTYPES
def test_large_layers_match_oracle(dtype):
    """Rows and columns longer than a warp, several CTAs per node."""
    pr, o, _ = _setup("wheel9", dtype, S=5, seed=7, shapes=LARGE)
    Harness(pr, o).run(3)


def test_messages_do_not_depend_on_the_grid():
    outs = []
    for grid in (0, 1, 3):
        pr, o, _ = _setup("wheel9", torch.float32, S=2, seed=3, shapes=LARGE)
        o.pg_grid = grid
        h = Harness(pr, o)
        for _ in range(3):
            h.eng.op.pg_mix()
            pr.fused.launch()
            h.eng.op.pg_step()
        torch.cuda.synchronize()
        outs.append(h.state())
    for s in outs[1:]:
        for key in ("theta", "vec", "pub"):
            assert np.array_equal(s[key], outs[0][key]), key


def test_graph_replay_equals_eager_launches():
    runs = []
    for capture in (False, True):
        pr, o, _ = _setup("wheel9", torch.float32, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        assert prog.launches_per_round() == 3 and prog.pr._metric_engine is None
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            states.append((_t(pr.arena.theta), _t(o.vec), _t(prog.eng.pub)))
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for x, y in zip(a, b):
            assert np.array_equal(x, y), f"round {k}"


def test_bytes_per_round_count_both_phases():
    pr, o, _ = _setup("cycle6", torch.float64)
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    lay = o.lay
    assert (lay.P, lay.Q, lay.B) == (9, 13, 9)
    b = eng.bytes_per_round()
    assert b["pulled_phase0"] == 12 * (9 + 9) * 8 and b["pulled_phase1"] == 12 * (13 + 9) * 8
    assert b["row"] == lay.width * 8 and b["pulled"] == (b["pulled_phase0"] + b["pulled_phase1"]) // 2


def test_capacity_is_refused():
    with pytest.raises(ValueError, match="at most 16 neighbors"):
        check_powergossip_capacity(17, 64, 8, 227 * 1024)
    with pytest.raises(ValueError, match="opt-in limit"):
        check_powergossip_capacity(16, 4096, 8, 227 * 1024)
    conf = {"alg_name": "powergossip", "alpha0": 0.05, "gamma": 1.0, "outer_iterations": 3}
    pr = PgProblem(nx.star_graph(17), torch.float32, 1, 0, SMALL, conf)
    o = PowerGossip(pr, DEV, conf)
    with pytest.raises(ValueError, match="powergossip handles at most 16 neighbors"):
        ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))


# ------------------------------------------------------------------------------------------ whole runs ----
PG = {"alg_name": "powergossip", "alpha0": 0.01, "mu": 0.001, "gamma": 1.0, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    return (PowerGossip(a, DEV, copy.deepcopy(conf)),
            PowerGossip(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch")))


def test_mnist_fp64_paper_shape_matches_torch_fp64():
    from test_gpu_mnist import _generic_problem
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=6, eval_every=3, conf=copy.deepcopy(PG))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=6, eval_every=3, conf=copy.deepcopy(PG))
    oa, ob = _pair(a, b, PG)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    oa._program.sync_back()
    r, rv, rm = _rel(a.arena.theta, b.arena.theta), _rel(oa.vec, ob.vec), _rel(oa.msg, ob.msg)
    print(f"\nMNIST fp64 powergossip: rel theta {r:.2e}, vec {rv:.2e}, msg {rm:.2e}")
    assert r < 1e-8 and rv < 1e-8 and rm < 1e-8
    assert a.forward_cnt == b.forward_cnt


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(PG))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(PG))
    oa, ob = _pair(a, b, PG)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64 powergossip: rel {r:.2e}")
    assert r < 1e-8
    oa._program.sync_back()
    assert _rel(oa.msg, ob.msg) < 1e-8 and _rel(oa.vec, ob.vec) < 1e-8


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(PG, outer_iterations=12)
        pr = _problem(5, 32, "fused", conf, M=100, eval_every=1000, graph=nx.wheel_graph(5))
        pr.conf["input_pipeline"] = pl
        opt = PowerGossip(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.msg.clone(), opt.vec.clone(), pr.forward_cnt))
    for x, y in zip(outs[0], outs[1]):
        assert torch.equal(x, y) if torch.is_tensor(x) else x == y


def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", dict(PG), graph=nx.cycle_graph(5), eval_every=3)
        opt = PowerGossip(pr, DEV, dict(PG))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.msg.clone(), opt.vec.clone()))
    for run in outs[1:]:
        for x, y in zip(run, outs[0]):
            assert torch.equal(x, y)


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    """Resume at round 3, which runs phase 1: the vectors and the messages come back from the checkpoint."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(PG, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(5, 32, "fused", conf, M=100, graph=nx.cycle_graph(5))
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = PowerGossip(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = PowerGossip(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = PowerGossip(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and torch.equal(o2.vec, o1.vec) and torch.equal(o2.msg, o1.msg)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.msg, of.msg) and torch.equal(o2.vec, of.vec)


def test_sequence_check_passes():
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        pr = _problem(6, 32, "fused", dict(PG), graph=nx.cycle_graph(6), eval_every=1000)
        c = dict(PG, debug_sequence_check=True, consensus_backend="auto" if backend == "fused" else "torch")
        opt = PowerGossip(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert opt._program.eng.seq_buf is not None
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
