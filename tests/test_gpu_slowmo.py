"""SlowMo on the fused sm_90a kernels: every ``slowmo_outer`` launch against the float64 oracle of
``tests/slowmo_oracle.py`` (|kernel - oracle| <= 16 err) on global and gossip rounds, in both dtypes, with and without the
base momentum row, on one-vector, padded and grid-stride rows (the round's other launches against their oracles in
``tests/pga_oracle.py``); sentinel rows left alone on gossip rounds and equal nodes after a global round; fused DSGD and
fused DSGDm with local momentum at a period past the run, bit for bit; whole fp64 runs against the PyTorch path; CUDA-graph
replay across the 64-round capture boundary; pipelines, determinism, checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import pga_oracle as po
import slowmo_oracle as so
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import MAX_ROUNDS_PER_GRAPH, RoundProgram
from nn_distributed_training_b200.optimizers import DSGD, DSGDm, GossipPGA, SlowMo
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
SM_GRAPHS = {k: v for k, v in GRAPHS.items() if k != "complete6_ptr"}
ROUNDS = 6
SENTINEL = 12345.0
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
GOSSIP = pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])
BASE = pytest.mark.parametrize("base", [0.0, 0.9], ids=["sgd", "momentum"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per launch and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:12s} {dt:5s} {r:.3f}")


def _setup(graph_key, dtype, S, n, period, gossip, base=0.0, n_pad=None, seed=0, equal_rows=False):
    conf = {"alg_name": "slowmo", "alpha0": 0.08, "mu": 2.0, "period": period, "gossip": gossip, "slow_momentum": 0.7,
            "slow_lr": 1.3, "base_momentum": base, "outer_iterations": ROUNDS, "profile": False}
    pr = KernelProblem(SM_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    th = torch.randn(1 if equal_rows else pr.N, n, generator=g, dtype=torch.float64)
    pr.arena.theta[:, :n] = th.expand(pr.N, n).to(dtype).to(DEV)
    o = SlowMo(pr, DEV, conf)
    # a nonzero slow momentum from the start, so beta_s u is exercised in the first global round
    u = 0.5 * torch.randn(1 if equal_rows else pr.N, n, generator=g, dtype=torch.float64)
    o.u[:, :n] = u.expand(pr.N, n).to(dtype).to(DEV)
    return pr, o


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def run_checked(pr, o, rounds=ROUNDS):
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert not eng.sum_mode and eng.C == 1
    u_T = co.unit_roundoff(NPDT[pr.dtype])
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    n, N = pr.n, pr.N
    src, op = pr.fused, eng.op
    rows = [o.anchor, o.u] + ([o.m] if o.m is not None else [])
    topos = [Topology(g) for g in pr.plan_graphs(o.oits, 0, 1)]
    tag = "outer_m" if o.m is not None else "outer"
    for k in range(rounds):
        glob, par = o.is_global(k), k & 1
        pub0, th0 = _t(eng.pub), _t(pr.arena.theta)
        op.pga_sum()
        op.pga_mix()
        torch.cuda.synchronize()
        th1 = _t(pr.arena.theta)
        if glob:
            s, es = po.pga_sum(pub0[par, 0, :N, :n])
        t = topos[k] if o.gossip else Topology(o.edgeless_graph())
        for l in range(N):
            want, err = po.pga_mix(l, th0[l, :n], pub0[par, 0, :N, :n], t.neighbors_noself, t.W, u_T, glob=glob,
                                   gossip=o.gossip, sums=(s, es) if glob else None)
            co.check(f"round {k} node {l} mix", th1[l, :n], want, err, C)
        saved = [r.clone() for r in rows]
        if not glob:        # a gossip round's slowmo_outer touches none of the rows
            for r in rows:
                r.fill_(SENTINEL)
        before = [_t(r) for r in rows]
        op.slowmo_outer()
        torch.cuda.synchronize()
        th2 = _t(pr.arena.theta)
        if not glob:
            assert np.array_equal(th2, th1), f"round {k}: a gossip round's slowmo_outer wrote theta"
            assert all(np.array_equal(_t(r), b) for r, b in zip(rows, before)), f"round {k}: a row was written"
            for r, v in zip(rows, saved):
                r.copy_(v)
        else:
            a0, u0 = before[0], before[1]
            gamma = float(eng.alpha[k - 1].item()) if k > 0 else float(NPDT[pr.dtype](o.alph0))
            a1, u1 = _t(o.anchor), _t(o.u)
            for l in range(N):
                un, eu, an, ea = so.slowmo_outer(th1[l, :n], a0[l, :n], u0[l, :n], gamma, o.slow_lr, o.slow_momentum,
                                                 u_T)
                WORST[(tag + "_u", dt)] = max(WORST[(tag + "_u", dt)],
                                              co.check(f"round {k} node {l} u", u1[l, :n], un, eu, C))
                WORST[(tag + "_a", dt)] = max(WORST[(tag + "_a", dt)],
                                              co.check(f"round {k} node {l} anchor", a1[l, :n], an, ea, C))
            assert np.array_equal(th2, a1), f"round {k}: theta is not the anchor"
            assert not a1[:, n:].any() and not u1[:, n:].any(), "padding of anchor / u"
            if o.m is not None:
                assert not o.m.any(), f"round {k}: m was not reset"
            if (a0 == a0[0]).all() and (u0 == u0[0]).all():
                assert (a1 == a1[0]).all() and (u1 == u1[0]).all() and (th2 == th2[0]).all(), f"round {k}"
        src.launch()
        torch.cuda.synchronize()
        gpart = _t(src.grad_part)
        (op.dsgd_step if o.m is None else op.dsgdm_step)()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == k + 1 and int(eng.done_ctr.item()) == 0
        th3, pub3 = _t(pr.arena.theta), _t(eng.pub)
        if o.m is None:
            alpha = float(eng.alpha[k].item())
            for l in range(N):
                want, err = po.dsgd_step(th2[l, :n], gpart[l, :, :n], alpha, u_T)
                co.check(f"round {k} node {l} step", th3[l, :n], want, err, C)
        assert np.array_equal(pub3[par ^ 1, 0, :N], th3)
    eng.check()
    return eng


# ------------------------------------------------------------------------------------------ per launch ----
@BASE
@GOSSIP
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(SM_GRAPHS))
def test_launches_match_oracle(graph_key, dtype, gossip, base):
    """Every graph (degrees 0-9, a changing graph), rows of 13 parameters (padding in the row), periods 2 and 3 (global
    rounds 1, 3, 5 or 2, 5), S rotating with the case."""
    i = sorted(SM_GRAPHS).index(graph_key)
    pr, o = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, 2 + i % 2, gossip, base, seed=i)
    run_checked(pr, o)


@BASE
@DTYPES
@pytest.mark.parametrize("period", [1, 4])
def test_every_round_global_and_one_global_round(period, dtype, base):
    """period 1: round 0 is global, with gamma = alpha0."""
    pr, o = _setup("star8", dtype, 5, 77, period, True, base, seed=period)
    run_checked(pr, o)


@BASE
@GOSSIP
@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype, gossip, base):
    """A row of exactly one vector, a padded row, and rows long enough that the grid is capped at the resident CTAs and
    every thread walks the row more than once."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o = _setup("random5to7", dtype, 5, vec, 2, gossip, base, n_pad=vec, seed=3)
    elif size == "padded":
        pr, o = _setup("random5to7", dtype, 3, 3 * vec + 1, 2, gossip, base, seed=5)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o = _setup("random5to7", dtype, 17, 140001, 2, gossip, base, seed=4)
        assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    run_checked(pr, o, rounds=4)


@BASE
@DTYPES
def test_nodes_bitwise_equal_after_a_global_round(dtype, base):
    """Equal rows and equal u on every node: anchors, u and theta stay bitwise equal across nodes after every global
    round (checked inside ``run_checked``)."""
    pr, o = _setup("wheel10", dtype, 4, 29, 2, True, base, seed=9, equal_rows=True)
    run_checked(pr, o)


# ------------------------------------------------------------------------------------------ whole runs ----
SC = {"alg_name": "slowmo", "alpha0": 0.01, "mu": 0.001, "period": 3, "slow_momentum": 0.5, "outer_iterations": 7,
      "profile": False}
DC = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 7, "profile": False}
MC = {"alg_name": "dsgdm", "alpha0": 0.01, "mu": 0.001, "beta": 0.9, "momentum": "local", "outer_iterations": 7,
      "profile": False}
# Whole fp64 runs against the PyTorch path: every launch is within 16 err of its oracle, a few units of 2^-53 of the
# values it touches, and the runs here are 7 rounds of 4 or 5 launches; 1e-10 leaves the gradients' amplification of
# those differences three orders of magnitude, the bound Gossip-PGA's whole runs use
WHOLE_RUN_REL = 1e-10


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = SlowMo(a, DEV, copy.deepcopy(conf))
    ob = SlowMo(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


@BASE
@GOSSIP
def test_mnist_fp64_paper_shape_matches_torch_fp64(gossip, base):
    from test_gpu_mnist import _generic_problem
    conf = dict(SC, gossip=gossip, base_momentum=base)
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64 (gossip {gossip}, base momentum {base}): rel {r:.2e}, anchor rel "
          f"{_rel(oa.anchor, ob.anchor):.2e}")
    assert r < WHOLE_RUN_REL and _rel(oa.anchor, ob.anchor) < WHOLE_RUN_REL
    assert a.forward_cnt == b.forward_cnt and oa.alph == ob.alph


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(SC))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(SC))
    oa, ob = _pair(a, b, SC)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64: rel {r:.2e}")
    assert r < WHOLE_RUN_REL
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


@pytest.mark.parametrize("nesterov", [False, True], ids=["heavy_ball", "nesterov"])
@BASE
@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_period_past_the_run_is_fused_dsgd_or_dsgdm_bit_for_bit(model, base, nesterov):
    if nesterov and not base:
        pytest.skip("nesterov applies to the base momentum")
    R = 12
    conf = dict(SC, period=R + 1, base_momentum=base, nesterov=nesterov, outer_iterations=R)
    oconf = dict(MC, nesterov=nesterov, outer_iterations=R) if base else dict(DC, outer_iterations=R)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem
        a, b = _problem(4, 32, "fused", conf, M=100), _problem(4, 32, "fused", oconf, M=100)
    else:
        from test_gpu_mlp_f64 import _density
        a, b = (_density(4, 500, M=700, opt_conf=copy.deepcopy(conf)),
                _density(4, 500, M=700, opt_conf=copy.deepcopy(oconf)))
    b.arena.theta.copy_(a.arena.theta)
    oa = SlowMo(a, DEV, copy.deepcopy(conf))
    ob = (DSGDm if base else DSGD)(b, DEV, copy.deepcopy(oconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    assert oa._program.launches_per_round() == ob._program.launches_per_round() + 2
    assert torch.equal(a.arena.theta, b.arena.theta)
    if base:
        assert torch.equal(oa.m, ob.m)


@pytest.mark.parametrize("period", [5, 7])
def test_graph_replay_across_the_capture_boundary_equals_eager_launches(period):
    from test_gpu_mnist import _problem
    R = MAX_ROUNDS_PER_GRAPH + 6
    outs = []
    for capture in (False, True):
        conf = dict(SC, period=period, base_momentum=0.9, outer_iterations=R)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100, eval_every=1000)
        pr.conf["input_pipeline"] = "resident"
        opt = SlowMo(pr, DEV, copy.deepcopy(conf))
        prog = opt._program = RoundProgram(opt)
        prog.capturable = capture
        assert prog.launches_per_round() == 5
        opt.run_rounds(R)
        torch.cuda.synchronize()
        assert bool(prog._graphs) == capture
        assert int(prog.eng.round_ctr.item()) == R
        prog.eng.check()
        outs.append((pr.arena.theta.clone(), opt.anchor.clone(), opt.u.clone(), opt.m.clone()))
    assert all(torch.equal(x, y) for x, y in zip(*outs))


@GOSSIP
@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline, gossip):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(SC, gossip=gossip, base_momentum=0.9, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = SlowMo(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.anchor.clone(), pr.forward_cnt, pr.calls.copy()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][2] == outs[1][2] and (outs[0][3] == outs[1][3]).all()


def test_bytes_per_round_are_gossip_pga_s():
    from test_gpu_mnist import _problem
    for gossip in (True, False):
        conf = dict(SC, gossip=gossip)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100)
        eng = RoundProgram(SlowMo(pr, DEV, copy.deepcopy(conf))).eng
        pconf = {k: v for k, v in conf.items() if k != "slow_momentum"}
        pq = _problem(5, 32, "fused", pconf, graph=nx.cycle_graph(5), M=100)
        peng = RoundProgram(GossipPGA(pq, DEV, dict(pconf, alg_name="gossip_pga"))).eng
        assert eng.bytes_per_round() == peng.bytes_per_round()
        row = pr.arena.n_pad * pr.arena.theta.element_size()
        assert eng.bytes_per_round()["pulled"] == (2 * 5 * row if gossip else 0)


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic():
    from test_gpu_mnist import _problem
    outs = []
    for _ in range(2):
        conf = dict(SC, base_momentum=0.9)
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = SlowMo(pr, DEV, copy.deepcopy(conf))
        opt.train()
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


@BASE
@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_global_round_is_bit_exact(tmp_path, model, base):
    """period 2: round 3 is global, so the resumed run starts with a global round at an odd k."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(SC, period=2, base_momentum=base, outer_iterations=7)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = SlowMo(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = SlowMo(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = SlowMo(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and o2.is_global(3)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.anchor, of.anchor) and torch.equal(o2.u, of.u)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt


@GOSSIP
def test_sequence_check_passes(gossip):
    """``debug_sequence_check``: every gossip-round pull reads a row tagged with its round; the fused run matches the
    PyTorch ops on the same fused forward/backward kernels."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(SC, gossip=gossip, debug_sequence_check=True,
                    consensus_backend="auto" if backend == "fused" else "torch")
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        opt = SlowMo(pr, DEV, copy.deepcopy(conf))
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            eng = opt._program.eng
            assert eng.seq_buf is not None
            torch.cuda.synchronize()
            assert int(eng.err.item()) == 0
            eng.check()
    _assert_mostly_close(outs[0], outs[1])
