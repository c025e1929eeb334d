"""SGP on the fused sm_90a kernels: ``sgp_mix`` and ``sgp_step`` one launch at a time against a float64 oracle
(|kernel - oracle| <= 16 u err), the push-sum weight tail bitwise equal to the weight every CTA divided by, then whole
runs against the PyTorch path, determinism, CUDA-graph replay, the input pipelines, checkpoint/resume and the sequence
check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
from test_gpu_consensus_kernels import KernelProblem
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import SGP
from nn_distributed_training_b200.utils.graph_generation import Topology, generate_from_conf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
ROUNDS, CHECKED = 6, (0, 1, 5)
S_LIST = [1, 4, 5, 16, 17]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:10s} {dt:5s} {r:.3f}")


def _gen(kind, N, **kw):
    return generate_from_conf(dict({"type": kind, "num_nodes": N}, **kw))[1]


def _source():
    """Node 0 sends to every other node and reads nobody (in-degree 0); the others form a directed ring."""
    g = nx.DiGraph()
    g.add_nodes_from(range(7))
    g.add_edges_from((0, i) for i in range(1, 7))
    g.add_edges_from((i, i % 6 + 1) for i in range(1, 7))
    return g


def _random_in_5_to_7():
    for seed in range(10000):
        g = nx.gnp_random_graph(10, 0.6, seed=seed, directed=True)
        d = [x for _, x in g.in_degree()]
        if min(d) == 5 and max(d) == 7 and nx.is_strongly_connected(g):
            return g
    raise AssertionError("no seed gives in-degrees 5..7")


# in-degrees 0-9 between them; a sequence of digraphs that changes every round
SGP_GRAPHS = {
    "source7": [_source()],                                   # 0 and 2
    "directed_cycle6": [_gen("directed_cycle", 6)],           # 1
    "exponential10": [_gen("exponential", 10)],               # 4
    "random_directed": [_random_in_5_to_7()],                 # 5-7
    "star9": [nx.star_graph(8)],                              # 1 and 8, undirected and irregular
    "wheel10": [nx.wheel_graph(10)],                          # 3 and 9
    "switch": [_gen("directed_cycle", 6), _gen("exponential", 6), nx.star_graph(5), _source().subgraph(range(6)).copy()],
}


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, S, n, n_pad=None, seed=0, far=True, oits=ROUNDS):
    conf = {"alg_name": "sgp", "alpha0": 0.08, "mu": 2.0, "outer_iterations": oits, "profile": False}
    pr = KernelProblem(SGP_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    th = torch.randn(pr.N, n, generator=g, dtype=torch.float64)
    pr.arena.theta[:, :n] = th.to(dtype).to(DEV)
    o = SGP(pr, DEV, conf)
    if far:        # push-sum weights far from 1 (as after many rounds on an irregular graph), theta = x / w
        o.w.copy_(torch.exp(2.0 * torch.randn(pr.N, generator=g, dtype=torch.float64)).to(DEV))
        o.x.copy_(pr.arena.theta * o.w.to(dtype).unsqueeze(1))
        pr.arena.theta.copy_(ref.sgp_debias(o.x, o.w))
    return pr, o, conf


def _state(pr, o, eng):
    L, n_pad = pr.N, pr.layout.n_pad
    t = lambda x: x.detach().double().cpu().numpy().copy()
    return dict(theta=t(pr.arena.theta), x=t(o.x), w=t(o.w), theta_t=pr.arena.theta.detach().cpu().clone(),
                x_t=o.x.detach().cpu().clone(), w_t=o.w.detach().cpu().clone(),
                pub=t(eng.pub[:, 0, :L, :n_pad]), pub_w=np.stack([t(eng.pub_weights(p)) for p in (0, 1)]),
                pub_tail=eng.pub[:, 0, :L].view(torch.uint8)[..., n_pad * eng.pub.element_size():].cpu().clone(),
                calls=pr.fused.calls.cpu().numpy().copy(), round_ctr=int(eng.round_ctr.item()),
                done_ctr=int(eng.done_ctr.item()), grad_part=t(pr.fused.grad_part))


class Harness:
    def __init__(self, pr, o):
        self.pr, self.o = pr, o
        self.graphs = pr.plan_graphs(o.oits, 0, 1)
        self.eng = ConsensusEngine(o, self.graphs)
        assert not self.eng.sum_mode
        assert self.eng.bytes_per_round()["row"] == pr.layout.n_pad * o.x.element_size() + 16
        self.dtype = pr.dtype
        self.npdt = NPDT[pr.dtype]
        self.u = co.unit_roundoff(self.npdt)
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.alpha = self.eng.alpha.cpu().double().numpy()
        self.n = pr.n

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        par, n = k & 1, self.n
        assert after["done_ctr"] == 0, name
        ends = name == "sgp_step"
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if ends else 0)), name
        for key in ("theta", "x"):
            assert not after[key][:, n:].any(), f"{name}: padding of {key} written"
        # every element of theta is x / w with the stored w: all CTAs of a node divided by the same bits
        assert torch.equal(after["theta_t"], ref.sgp_debias(after["x_t"], after["w_t"])), f"{name} round {k}: theta != x / w"
        key = (name, self.dt)
        if name == "sgp_mix":
            assert np.array_equal(after["pub"], before["pub"]) and torch.equal(after["pub_tail"], before["pub_tail"])
            if not check:
                return
            A = Topology(self.graphs[k]).push_weights.astype(self.npdt).astype(np.float64)   # the kernel's weights
            nbrs = Topology(self.graphs[k]).neighbors_noself
            xs, ws = before["pub"][par], before["pub_w"][par]
            x = np.zeros_like(xs)
            e_x = np.zeros_like(xs)
            w = np.zeros(self.pr.N)
            e_w = np.zeros(self.pr.N)
            for i in range(self.pr.N):
                x[i], e_x[i] = co._mix(i, before["x"][i], xs, nbrs, A, self.u)
                wi, mag = A[i, i] * ws[i], abs(A[i, i] * ws[i])
                for j in nbrs[i]:
                    wi += A[i, j] * ws[j]
                    mag += abs(A[i, j] * ws[j])
                w[i], e_w[i] = wi, co.U64 * (mag + abs(wi))
            th = x / w[:, None]
            e_th = (e_x + np.abs(th) * e_w[:, None]) / w[:, None] + 2 * self.u * np.abs(th)
            WORST[key] = max(WORST[key], co.check(f"{name} round {k} w", after["w"], w, e_w, C),
                             co.check(f"{name} round {k} x", after["x"], x, e_x, C),
                             co.check(f"{name} round {k} theta", after["theta"], th, e_th, C))
            return
        # sgp_step
        assert torch.equal(after["w_t"], before["w_t"]), "sgp_step wrote w"
        assert np.array_equal(after["pub"][par], before["pub"][par]), "sgp_step wrote the parity being read"
        assert torch.equal(after["pub_tail"][par], before["pub_tail"][par])
        assert np.array_equal(after["pub"][par ^ 1], after["x"]), f"{name} round {k}: published x"
        assert np.array_equal(after["pub_w"][par ^ 1], after["w"]), f"{name} round {k}: published w"
        if not check:
            return
        g, e_g = co.sum_partials(before["grad_part"], self.u)
        a = self.alpha[k]
        x = before["x"] - a * g
        e_x = a * e_g + self.u * (np.abs(before["x"]) + 2.0 * a * np.abs(g))
        WORST[key] = max(WORST[key], co.check(f"{name} round {k} x", after["x"], x, e_x, C))

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            self.launch("sgp_mix", op.sgp_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("sgp_step", op.sgp_step, k, check=chk)
        self.eng.check()


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(SGP_GRAPHS))
def test_launches_match_oracle(graph_key, dtype):
    """In-degrees 0-9, a graph that changes every round, rows of 77 parameters padded to the row alignment, S rotating
    with the case, push-sum weights far from 1."""
    i = sorted(SGP_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], n=77, seed=i)
    Harness(pr, o).run()


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8 (degree-9 hub: both neighbor groups)."""
    pr, o, conf = _setup("wheel10", dtype, S, n=100, seed=S, far=S % 2 == 0)
    Harness(pr, o).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("size", ["one_unit", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    """A row shorter than a CTA's span, and rows long enough that the grid is capped at the resident CTAs and every
    node has many CTAs, all of which must agree on w."""
    if size == "one_unit":
        pr, o, conf = _setup("random_directed", dtype, 5, n=128, seed=3)
        Harness(pr, o).run()
        return
    pr, o, conf = _setup("exponential10", dtype, 17, n=140001, seed=4)
    Harness(pr, o).run(rounds=2, checked=(0, 1))


@DTYPES
def test_graph_replay_equals_eager_launches(dtype):
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup("switch", dtype, 5, n=300, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            s = _state(pr, o, prog.eng)
            states.append({k: v for k, v in s.items() if isinstance(v, np.ndarray)})
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            assert np.array_equal(x, b[key]), f"round {k}: {key}"


# ------------------------------------------------------------------------------------------ whole runs ----
SG = {"alg_name": "sgp", "alpha0": 0.05, "mu": 0.01, "outer_iterations": 7, "profile": False}
EXPO5 = _gen("exponential", 5)


def _rdg(N):
    """A strongly connected, irregular digraph: w moves away from 1.  (A node without in-neighbors would lose its mass
    every round and blow its gradient steps up by 1 / w; whole runs train on strongly connected graphs.)"""
    return _gen("random_directed", N, p=0.5, seed=1, gen_attempts=100)


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _mnist64(conf, backend):
    from test_gpu_mnist import _generic_problem
    pr = _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    pr.graph = pr._base_graph = _rdg(5)
    return pr


def _density64(conf, backend):
    from test_gpu_mlp_f64 import _density
    pr = _density(4, 500, M=700, backend=backend, opt_conf=copy.deepcopy(conf))
    pr.graph = pr._base_graph = _rdg(4)
    return pr


@pytest.mark.parametrize("model", ["mnist_paper_fp64", "density_fp64"])
def test_fp64_runs_match_torch_path(model):
    make = _mnist64 if model == "mnist_paper_fp64" else _density64
    a, b = make(SG, "fused"), make(SG, "torch")
    b.arena.theta.copy_(a.arena.theta)
    oa = SGP(a, DEV, copy.deepcopy(SG))
    ob = SGP(b, DEV, dict(copy.deepcopy(SG), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    assert (oa.w - 1.0).abs().max() > 1e-2
    assert torch.isfinite(a.arena.theta).all()
    for name, x, y in (("theta", a.arena.theta, b.arena.theta), ("x", oa.x, ob.x), ("w", oa.w, ob.w)):
        r = _rel(x, y)
        print(f"{model} {name}: rel {r:.2e}")
        assert r < 1e-13, name
    assert a.forward_cnt == b.forward_cnt


def test_online_density_fp64_dynamic_graph_matches_torch_fp64(tmp_path):
    """The online problem (graph planned from the robot poses, changing over the run) in float64: push-sum needs no
    rebuild of a doubly stochastic matrix when the graph changes."""
    from test_gpu_mlp_f64 import _online_problem
    oc = dict(SG, alpha0=0.002, outer_iterations=9)
    fused = _online_problem("fused", str(tmp_path), oc)
    refp = _online_problem("torch", str(tmp_path), oc)
    refp.arena.theta.copy_(fused.arena.theta)
    of = SGP(fused, DEV, copy.deepcopy(oc))
    orf = SGP(refp, DEV, dict(copy.deepcopy(oc), consensus_backend="torch"))
    orf.train()
    of.train()
    assert len(of._program.eng.topos) > 1
    assert (fused.positions() == refp.positions()).all()
    assert fused.forward_cnt == refp.forward_cnt
    for key in ("validation_loss", "train_loss_moving_average"):
        torch.testing.assert_close(fused.metrics[key][-1], refp.metrics[key][-1], rtol=1e-9, atol=1e-12)
    for name, x, y in (("theta", fused.arena.theta, refp.arena.theta), ("w", of.w, orf.w)):
        r = _rel(x, y)
        print(f"online density {name}: rel {r:.2e}")
        assert r < 1e-13, name


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", copy.deepcopy(SG), graph=EXPO5, eval_every=3)
        opt = SGP(pr, DEV, copy.deepcopy(SG))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.x.clone(), opt.w.clone()))
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0]))


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(SG, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, graph=_rdg(4), eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = SGP(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        opt._program.sync_back()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.x.clone(), opt.w.clone(), pr.forward_cnt))
        assert torch.isfinite(pr.arena.theta).all() and not torch.all(opt.w == 1.0)
    assert all(torch.equal(x, y) for x, y in zip(outs[0][:3], outs[1][:3]))
    assert outs[0][3] == outs[1][3]


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(SG, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100, graph=_rdg(4))
    else:
        def make():
            return _density64(conf, "fused")
    full = make()
    of = SGP(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = SGP(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3 and not torch.all(o1.w == 1.0)
    second = make()
    o2 = SGP(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and torch.equal(o2.x, o1.x) and torch.equal(o2.w, o1.w)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.x, of.x) and torch.equal(o2.w, of.w)
    assert o2.alph == of.alph
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_on_an_sgp_run():
    """``debug_sequence_check``: every in-neighbor row read is tagged with the current round."""
    from test_gpu_mnist import _problem
    conf = dict(SG, debug_sequence_check=True, outer_iterations=10)
    pr = _problem(6, 32, "fused", conf, graph=_gen("exponential", 6), eval_every=1000)
    opt = SGP(pr, DEV, conf)
    opt.train()
    assert opt._program.eng.seq_buf is not None
    opt._program.eng.check()
