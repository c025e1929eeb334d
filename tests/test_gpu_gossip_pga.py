"""Gossip-PGA on the fused sm_90a kernels: every ``pga_sum`` / ``pga_mix`` / ``dsgd_step`` launch against the float64
oracle of ``tests/pga_oracle.py`` (|kernel - oracle| <= 16 err) on global and gossip rounds, with gossip and as local SGD;
the sum buffer left alone on gossip rounds and equal rows after a global mix; fused DSGD at a period past the run and
fused complete-graph DSGD in sum mode at period 1, bit for bit; whole fp64 runs against the PyTorch path; CUDA-graph
replay across the 64-round capture boundary; pipelines, determinism, checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import pga_oracle as po
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import MAX_ROUNDS_PER_GRAPH, RoundProgram
from nn_distributed_training_b200.optimizers import DSGD, GossipPGA
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# degrees 0..16: isolated (0..3), path2 (1), cycle6 (2), random (5..7), complete6 (5, through the pointer table: a
# complete base graph is no sum mode for gossip_pga), star8 (hub 8), wheel10 (hub 9), star16 (hub 16), a changing graph
PGA_GRAPHS = {k: v for k, v in GRAPHS.items() if k != "complete6_ptr"}
PGA_GRAPHS["star16"] = [nx.star_graph(16)]
ROUNDS = 6
SENTINEL = 12345.0
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
GOSSIP = pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per launch and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:12s} {dt:5s} {r:.3f}")


def _setup(graph_key, dtype, S, n, period, gossip, n_pad=None, seed=0):
    conf = {"alg_name": "gossip_pga", "alpha0": 0.08, "mu": 2.0, "period": period, "gossip": gossip,
            "outer_iterations": ROUNDS, "profile": False}
    pr = KernelProblem(PGA_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, GossipPGA(pr, DEV, conf)


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def run_checked(pr, o, rounds=ROUNDS):
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert not eng.sum_mode and eng.C == 1
    u = co.unit_roundoff(NPDT[pr.dtype])
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    n, N = pr.n, pr.N
    src, op = pr.fused, eng.op
    eng.sum_buf.local.fill_(SENTINEL)
    topos = [Topology(g) for g in pr.plan_graphs(o.oits, 0, 1)]
    for k in range(rounds):
        glob, par, sp = o.is_global(k), k & 1, (k // o.period) & 1
        pub0, th0, sum0 = _t(eng.pub), _t(pr.arena.theta), _t(eng.sum_buf.local)
        op.pga_sum()
        torch.cuda.synchronize()
        sum1 = _t(eng.sum_buf.local)
        if glob:
            s, es = po.pga_sum(pub0[par, 0, :N, :n])
            WORST[("pga_sum", dt)] = max(WORST[("pga_sum", dt)], co.check(f"round {k} sum", sum1[sp, 0, :n], s, es, C))
            assert not sum1[sp, 0, n:].any(), "padding of the partial sum"
            assert np.array_equal(sum1[sp ^ 1], sum0[sp ^ 1]), "the other global round's buffer was written"
        else:
            assert np.array_equal(sum1, sum0), f"round {k}: a gossip round's pga_sum wrote the sum buffer"
        op.pga_mix()
        torch.cuda.synchronize()
        th1 = _t(pr.arena.theta)
        if glob:
            assert (th1 == th1[0]).all(), f"round {k}: rows differ after the global mix"
        t = topos[k] if o.gossip else Topology(o.edgeless_graph())
        for l in range(N):
            want, err = po.pga_mix(l, th0[l, :n], pub0[par, 0, :N, :n], t.neighbors_noself, t.W, u, glob=glob,
                                   gossip=o.gossip, sums=(s, es) if glob else None)
            key = "mix_global" if glob else ("mix_gossip" if o.gossip else "mix_local")
            WORST[(key, dt)] = max(WORST[(key, dt)], co.check(f"round {k} node {l} mix", th1[l, :n], want, err, C))
        assert not th1[:, n:].any(), "padding of theta"
        src.launch()
        torch.cuda.synchronize()
        gpart = _t(src.grad_part)
        op.dsgd_step()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == k + 1 and int(eng.done_ctr.item()) == 0
        th2, pub2 = _t(pr.arena.theta), _t(eng.pub)
        alpha = float(eng.alpha[k].item())
        for l in range(N):
            want, err = po.dsgd_step(th1[l, :n], gpart[l, :, :n], alpha, u)
            WORST[("step", dt)] = max(WORST[("step", dt)], co.check(f"round {k} node {l} step", th2[l, :n], want, err, C))
        assert np.array_equal(pub2[par ^ 1, 0, :N], th2)
    eng.check()
    return eng


# ------------------------------------------------------------------------------------------ per launch ----
@GOSSIP
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(PGA_GRAPHS))
def test_launches_match_oracle(graph_key, dtype, gossip):
    """Every graph (degrees 0-16, a changing graph), rows of 13 parameters (padding in the row), periods 2 and 3 (global
    rounds 1, 3, 5 or 2, 5: both partial-sum buffers), S rotating with the case."""
    i = sorted(PGA_GRAPHS).index(graph_key)
    pr, o = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, 2 + i % 2, gossip, seed=i)
    eng = run_checked(pr, o)
    assert eng.dmax == (1 if not gossip else max(1, max(Topology(g).max_degree for g in PGA_GRAPHS[graph_key])))


@DTYPES
@pytest.mark.parametrize("period", [1, 4])
def test_every_round_global_and_one_global_round(period, dtype):
    pr, o = _setup("star16", dtype, 5, 77, period, True, seed=period)
    run_checked(pr, o)


@GOSSIP
@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype, gossip):
    """A row of exactly one vector, a padded row, and rows long enough that the mix's grid is capped at the resident
    CTAs and every thread walks the row more than once."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o = _setup("random5to7", dtype, 5, vec, 2, gossip, n_pad=vec, seed=3)
    elif size == "padded":
        pr, o = _setup("random5to7", dtype, 3, 3 * vec + 1, 2, gossip, seed=5)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o = _setup("random5to7", dtype, 17, 140001, 2, gossip, seed=4)
        assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    run_checked(pr, o, rounds=4)


# ------------------------------------------------------------------------------------------ whole runs ----
PC = {"alg_name": "gossip_pga", "alpha0": 0.01, "mu": 0.001, "period": 3, "outer_iterations": 7, "profile": False}
DC = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = GossipPGA(a, DEV, copy.deepcopy(conf))
    ob = GossipPGA(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


@GOSSIP
def test_mnist_fp64_paper_shape_matches_torch_fp64(gossip):
    from test_gpu_mnist import _generic_problem
    conf = dict(PC, gossip=gossip)
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64 (gossip {gossip}): rel {r:.2e}")
    assert r < 1e-10
    assert a.forward_cnt == b.forward_cnt and oa.alph == ob.alph


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(PC))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(PC))
    oa, ob = _pair(a, b, PC)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64: rel {r:.2e}")
    assert r < 1e-10
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_period_past_the_run_is_fused_dsgd_bit_for_bit(model):
    R = 12
    conf, dconf = dict(PC, period=R + 1, outer_iterations=R), dict(DC, outer_iterations=R)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem
        a, b = _problem(4, 32, "fused", conf, M=100), _problem(4, 32, "fused", dconf, M=100)
    else:
        from test_gpu_mlp_f64 import _density
        a, b = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf)), _density(4, 500, M=700, opt_conf=copy.deepcopy(dconf))
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = GossipPGA(a, DEV, copy.deepcopy(conf)), DSGD(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    assert oa._program.launches_per_round() == ob._program.launches_per_round() + 1
    assert torch.equal(a.arena.theta, b.arena.theta)


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_period_one_is_fused_complete_graph_dsgd_in_sum_mode_bit_for_bit(model):
    R = 12
    conf, dconf = dict(PC, period=1, outer_iterations=R), dict(DC, outer_iterations=R)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem
        a = _problem(4, 32, "fused", conf, M=100, graph=nx.cycle_graph(4))
        b = _problem(4, 32, "fused", dconf, M=100, graph=nx.complete_graph(4))
    else:
        from test_gpu_mlp_f64 import _density
        a, b = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf)), _density(4, 500, M=700, opt_conf=copy.deepcopy(dconf))
        b.graph = b._base_graph = nx.complete_graph(4)
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = GossipPGA(a, DEV, copy.deepcopy(conf)), DSGD(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert ob._program.eng.sum_mode and not oa._program.eng.sum_mode
    assert torch.equal(a.arena.theta, b.arena.theta)


@pytest.mark.parametrize("period", [5, 7])
def test_graph_replay_across_the_capture_boundary_equals_eager_launches(period):
    from test_gpu_mnist import _problem
    R = MAX_ROUNDS_PER_GRAPH + 6
    outs = []
    for capture in (False, True):
        conf = dict(PC, period=period, outer_iterations=R)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100, eval_every=1000)
        pr.conf["input_pipeline"] = "resident"
        opt = GossipPGA(pr, DEV, copy.deepcopy(conf))
        prog = opt._program = RoundProgram(opt)
        prog.capturable = capture
        assert prog.launches_per_round() == 4
        opt.run_rounds(R)
        torch.cuda.synchronize()
        assert bool(prog._graphs) == capture
        assert int(prog.eng.round_ctr.item()) == R
        prog.eng.check()
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


@GOSSIP
@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline, gossip):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(PC, gossip=gossip, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = GossipPGA(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), pr.forward_cnt, pr.calls.copy()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()


def test_bytes_per_round():
    from test_gpu_mnist import _problem
    for gossip in (True, False):
        conf = dict(PC, gossip=gossip)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100)
        opt = GossipPGA(pr, DEV, copy.deepcopy(conf))
        eng = RoundProgram(opt).eng
        b = eng.bytes_per_round()
        row = pr.arena.n_pad * pr.arena.theta.element_size()
        assert b == {"row": row, "pulled": 2 * 5 * row if gossip else 0, "global_row": pr.arena.n_pad * 8, "period": 3}


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic():
    from test_gpu_mnist import _problem
    outs = []
    for _ in range(2):
        pr = _problem(5, 32, "fused", PC, graph=nx.wheel_graph(5), eval_every=3)
        opt = GossipPGA(pr, DEV, copy.deepcopy(PC))
        opt.train()
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    """period 2: round 3 is global, so the resumed run starts with a global round at an odd k."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(PC, period=2, outer_iterations=7)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = GossipPGA(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = GossipPGA(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = GossipPGA(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and o2.is_global(3)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt


@GOSSIP
def test_sequence_check_passes(gossip):
    """``debug_sequence_check``: every gossip-round pull reads a row tagged with its round; the fused run matches the
    PyTorch ops on the same fused forward/backward kernels."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(PC, gossip=gossip, debug_sequence_check=True,
                    consensus_backend="auto" if backend == "fused" else "torch")
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        opt = GossipPGA(pr, DEV, copy.deepcopy(conf))
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            eng = opt._program.eng
            assert eng.seq_buf is not None
            torch.cuda.synchronize()
            assert int(eng.err.item()) == 0
            eng.check()
    _assert_mostly_close(outs[0], outs[1])
