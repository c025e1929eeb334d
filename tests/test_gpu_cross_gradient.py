"""Cross-gradient gossip on the fused sm_90a kernels: ``xg_pull``, ``xg_publish`` and ``xg_step`` one launch at a time
against the float64 oracle with the bound of ``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err); the cross
points byte-equal to the neighbors' rows, NaN in the unread channels; the cross-point forward/backward of every
training kernel at the own row (bit for bit) in the resident, staged and host pipelines; the draw counters; the
node order; whole runs against the PyTorch path and against fused local SGD; CUDA-graph replay, determinism,
checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import xg_oracle as xo
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, GradSource, KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import MAX_ROUNDS_PER_GRAPH, RoundProgram
from nn_distributed_training_b200.optimizers import CrossGradient, DSGD, GossipPGA
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


def _star_of(deg):
    return nx.star_graph(deg) if deg > 0 else nx.empty_graph(3)


# degrees 0..9 and 16 at a hub (the leaves have degree 1), and the fixed graphs of the consensus kernel tests
XG_GRAPHS = {f"star{d}": [_star_of(d)] for d in list(range(10)) + [16]}
XG_GRAPHS.update({k: v for k, v in GRAPHS.items() if len(v) == 1 and not k.endswith("_sum")})
ROUNDS = 3


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per output and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:22s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
class CrossSource(GradSource):
    """GradSource with one more set of partials per cross slot (other seeded values, the same draw counter)."""

    def __init__(self, L, S, n, n_pad, dtype, seed):
        super().__init__(L, S, n, n_pad, dtype, seed)
        self.args = (L, S, n, n_pad, dtype, seed)
        self.cross = []

    def enable_cross_points(self, theta_x):
        L, S, n, n_pad, dtype, seed = self.args
        self.cross = [GradSource(L, S, n, n_pad, dtype, seed + 1000 + e) for e in range(theta_x.shape[0])]
        self.grad_part_x = torch.zeros(theta_x.shape[0], L, S, n_pad, dtype=dtype, device=DEV)

    def launch_cross(self, e):
        src = self.cross[e]
        src.calls.copy_(self.calls)
        src.launch()
        self.grad_part_x[e].copy_(src.grad_part)


class CrossProblem(KernelProblem):
    def __init__(self, graphs, n, dtype, S, seed=0, n_pad=None, conf=None):
        super().__init__(graphs, n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
        self.fused = CrossSource(self.N, S, n, self.layout.n_pad, dtype, seed)
        self.fused.pr_calls = self.calls


def _setup(graph_key, dtype, S, n, lam, n_pad=None, seed=0):
    conf = {"alg_name": "cross_gradient", "alpha0": 0.08, "mu": 0.5, "cross_weight": lam, "outer_iterations": ROUNDS,
            "profile": False, "complete_graph_mode": "sum"}
    pr = CrossProblem(XG_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, CrossGradient(pr, DEV, conf)


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def run_checked(pr, o, rounds=ROUNDS, nan_unread=False):
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert eng.C == 1 + o.dmax and not eng.sum_mode and eng.rounds_per_step == 2
    u = co.unit_roundoff(NPDT[pr.dtype])
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    n, N = pr.n, pr.N
    src, op = pr.fused, eng.op
    tp = Topology(pr.graph)
    W, nb, rs = tp.W, tp.neighbors_noself, tp.reverse_slots()
    alphas = o.alpha_table(rounds)
    for k in range(rounds):
        p = 2 * k
        pub0, th = _t(eng.pub), _t(pr.arena.theta)
        if nan_unread:        # the cross channels no step reads: the idle slots of both parities
            for i in range(N):
                eng.pub[:, 1 + len(nb[i]):, i] = float("nan")
        op.xg_pull()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == p
        xmix, tx = _t(eng.xmix), _t(o.theta_x)
        for i in range(N):
            for e in range(o.dmax):
                want = pub0[0, 0, nb[i][e]] if e < len(nb[i]) else th[i]
                assert np.array_equal(tx[e, i], want), (k, i, e)      # byte copies (NaN never appears here)
            m, em = xo.mix(th[i, :n], W[i, i], [W[i, j] for j in nb[i]], [pub0[0, 0, j, :n] for j in nb[i]], u)
            WORST[("xmix", dt)] = max(WORST[("xmix", dt)], co.check(f"round {k} node {i} xmix", xmix[i, :n], m, em, C))
        src.launch()
        for e in range(o.dmax):
            src.launch_cross(e)
        torch.cuda.synchronize()
        gpart, gx, calls0 = _t(src.grad_part), _t(src.grad_part_x), src.calls.cpu().numpy().copy()
        op.xg_publish()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == p + 1 and int(eng.done_ctr.item()) == 0
        assert np.array_equal(src.calls.cpu().numpy(), calls0), "xg_publish advanced the draw counters"
        pub1, g = _t(eng.pub), _t(eng.xg_g)
        for i in range(N):
            want, eg = xo.partial_sum(gpart[i, :, :n], u)
            WORST[("g", dt)] = max(WORST[("g", dt)], co.check(f"round {k} node {i} g", g[i, :n], want, eg, C))
            for e in range(len(nb[i])):
                want, eg = xo.partial_sum(gx[e, i, :, :n], u)
                r = co.check(f"round {k} node {i} slot {e}", pub1[1, 1 + e, i, :n], want, eg, C)
                WORST[("cross", dt)] = max(WORST[("cross", dt)], r)
        assert np.array_equal(pub1[0], pub0[0]) or nan_unread, "xg_publish wrote the round's own parity"
        op.xg_step()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == p + 2
        assert np.array_equal(src.calls.cpu().numpy(), calls0 + 1)
        pub2, th2 = _t(eng.pub), _t(pr.arena.theta)
        assert np.array_equal(pub2[0, 0, :N], th2)
        assert not np.isnan(th2).any()
        for i in range(N):
            recv = [pub1[1, 1 + rs[i][e], j, :n] for e, j in enumerate(nb[i])]
            x, ex = xo.step(xmix[i, :n], g[i, :n], float(o.coef0[i]), [float(o.coef[i, e]) for e in range(len(nb[i]))],
                            recv, NPDT[pr.dtype](alphas[k]), u)
            WORST[("theta", dt)] = max(WORST[("theta", dt)], co.check(f"round {k} node {i} theta", th2[i, :n], x, ex, C))
            assert not th2[i, n:].any(), "padding written"
    eng.check()
    return eng


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(XG_GRAPHS))
def test_launches_match_oracle(graph_key, dtype):
    """Hub degrees 0..9 and 16 and the fixed graphs of the consensus kernel tests (the complete graph through the
    pointer table), rows of 13 parameters, S and lam rotating with the case."""
    i = sorted(XG_GRAPHS).index(graph_key)
    pr, o = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, (1.0, 0.5, 0.3, 0.0)[i % 4], seed=i)
    run_checked(pr, o)


@DTYPES
@pytest.mark.parametrize("S", [1, 3, 5, 17])
def test_every_partial_count_matches_oracle(S, dtype):
    pr, o = _setup("star16", dtype, S, 77, 0.7, seed=S)
    run_checked(pr, o, rounds=2)


@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o = _setup("random5to7", dtype, 5, vec, 0.6, n_pad=vec, seed=3)
    elif size == "padded":
        pr, o = _setup("random5to7", dtype, 3, 3 * vec + 1, 0.6, seed=5)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o = _setup("random5to7", dtype, 4, 140001, 0.6, seed=4)
        assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    run_checked(pr, o, rounds=2)


@DTYPES
def test_nan_in_unread_cross_channels_changes_no_bit(dtype):
    outs = []
    for nan in (False, True):
        pr, o = _setup("star5", dtype, 3, 29, 0.8, seed=11)
        run_checked(pr, o, rounds=2, nan_unread=nan)
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


# -------------------------------------------------------------------- cross-point forward/backward ----
XC = {"alg_name": "cross_gradient", "alpha0": 0.01, "mu": 0.001, "cross_weight": 0.5, "outer_iterations": 7,
      "profile": False}
KERNELS = ["fp64_cluster", "fp32_cluster", "batch_split", "generic", "mlp_bf16", "mlp_fp64"]


def _mnist(kind, backend="fused", conf=None, graph=None):
    from test_gpu_mnist import _generic_problem, _problem
    conf = copy.deepcopy(conf or XC)
    if kind == "fp64_cluster":
        return _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=5, conf=conf)
    if kind == "fp32_cluster":
        return _problem(4, 32, backend, conf, M=100, **({"graph": graph} if graph is not None else {}))
    if kind == "batch_split":
        return _problem(4, 96, backend, conf, M=200)
    return _generic_problem((4, 3, 32), torch.float32, backend, B=32, N=4, conf=conf)      # generic conv net


def _mlp(kind, conf=None):
    if kind == "mlp_bf16":
        from test_gpu_mlp import _density_problem
        return _density_problem("fused", B=500, M=1500, N=4)
    from test_gpu_mlp_f64 import _density
    return _density(4, 500, M=700, opt_conf=copy.deepcopy(conf or XC))


@pytest.mark.parametrize("kind", KERNELS)
def test_cross_points_at_theta_equal_the_own_point_bit_for_bit(kind):
    """Property 6: every cross point at the node's own row gives the own partials bit for bit, twice in a row (the draw
    counters of every op advance together)."""
    pr = _mnist(kind) if kind in KERNELS[:4] else _mlp(kind)
    fz = pr.fused
    o = CrossGradient(pr, DEV, copy.deepcopy(XC))
    assert len(fz.cross) == o.dmax >= 1
    o.theta_x.copy_(pr.arena.theta.unsqueeze(0).expand_as(o.theta_x))
    # the bf16 MLP kernel adds the output layer's w4 and b4 gradients with shared-memory float atomics (GT-HSGD's
    # exception): bit for bit up to them, to float32 summation order on them
    atomics = kind == "mlp_bf16"
    cut = pr.layout.slots[-2].offset if atomics else pr.arena.n_pad
    for _ in range(2):
        fz.launch()
        for e in range(o.dmax):
            fz.launch_cross(e)
        torch.cuda.synchronize()
        for e in range(o.dmax):
            assert torch.equal(fz.grad_part[..., :cut], fz.grad_part_x[e][..., :cut]), e
            if atomics:
                torch.testing.assert_close(fz.grad_part, fz.grad_part_x[e], rtol=1e-5, atol=1e-7)
        assert fz.grad_part.abs().sum() > 0
        if kind in KERNELS[:4]:
            for pt in fz.cross:
                assert torch.equal(fz.calls, pt["calls"])
        else:
            fz.calls += 1           # the consensus step's bookkeeping
    print(f"\n{kind}: {getattr(fz, 'kernel_name', type(fz).__name__)}")


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_cross_point_direct_ops_read_the_staged_batch(pipeline):
    pr = _mnist("fp32_cluster")
    pr.conf["input_pipeline"] = pipeline
    o = CrossGradient(pr, DEV, copy.deepcopy(XC))
    prog = o._program = RoundProgram(o)
    assert prog.pipeline == pipeline and prog.launches_per_round() == 5 + o.dmax     # staging, 3 + (1 + dmax)
    fz = pr.fused
    o.theta_x.copy_(pr.arena.theta.unsqueeze(0).expand_as(o.theta_x))
    for b in (0, 1):
        fz.gather_ops[b].launch()
        fz.direct_ops[b][0].train()
        for pt in fz.cross:
            pt["direct"][b].train()
        torch.cuda.synchronize()
        for e, pt in enumerate(fz.cross):
            assert torch.equal(fz.grad_part, fz.grad_part_x[e]), (b, e)
            assert torch.equal(fz.calls, pt["calls"])


@pytest.mark.parametrize("pipeline", ["resident", "staged", "host"])
def test_draw_counters_equal_dsgd(pipeline):
    """After a round every draw counter (the training op's and each cross op's twin) equals DSGD's."""
    outs = []
    for alg in ("cross_gradient", "dsgd"):
        conf = dict(XC, outer_iterations=12) if alg == "cross_gradient" else \
            {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 12}
        pr = _mnist("fp32_cluster", conf=conf)
        pr.conf["input_pipeline"] = pipeline
        o = (CrossGradient if alg == "cross_gradient" else DSGD)(pr, DEV, copy.deepcopy(conf))
        o.run_rounds(5)
        o.run_rounds(4)
        torch.cuda.synchronize()
        outs.append((pr, o))
    (pa, oa), (pb, ob) = outs
    assert (pa.calls == pb.calls).all() and (pa.calls == 9).all() and pa.forward_cnt == pb.forward_cnt
    assert torch.equal(pa.fused.calls, pb.fused.calls)
    for pt in pa.fused.cross:
        assert torch.equal(pt["calls"], pb.fused.calls)


# ------------------------------------------------------------------------------------------ whole runs ----
def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def test_mnist_fp64_paper_shape_matches_torch_fp64():
    from test_gpu_mnist import _generic_problem
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(XC))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(XC))
    b.arena.theta.copy_(a.arena.theta)
    oa = CrossGradient(a, DEV, copy.deepcopy(XC))
    ob = CrossGradient(b, DEV, dict(copy.deepcopy(XC), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64: rel {r:.2e}")
    assert r < 1e-12
    assert a.forward_cnt == b.forward_cnt


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(XC))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(XC))
    b.arena.theta.copy_(a.arena.theta)
    oa = CrossGradient(a, DEV, copy.deepcopy(XC))
    ob = CrossGradient(b, DEV, dict(copy.deepcopy(XC), consensus_backend="torch"))
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64: rel {r:.2e}")
    assert r < 1e-12
    assert a.forward_cnt == b.forward_cnt


@pytest.mark.parametrize("lam", [0.0, 0.5, 1.0])
def test_edgeless_graph_is_fused_local_sgd_bit_for_bit(lam):
    """Property 2 on the fused kernels: the edgeless graph equals fused Gossip-PGA local SGD with a period past the
    run."""
    from test_gpu_mnist import _problem
    R = 10
    xc = dict(XC, cross_weight=lam, outer_iterations=R)
    pc = {"alg_name": "gossip_pga", "alpha0": XC["alpha0"], "mu": XC["mu"], "period": R + 1, "gossip": False,
          "outer_iterations": R, "profile": False}
    a = _problem(4, 32, "fused", xc, graph=nx.empty_graph(4), M=100)
    b = _problem(4, 32, "fused", pc, graph=nx.cycle_graph(4), M=100)
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = CrossGradient(a, DEV, copy.deepcopy(xc)), GossipPGA(b, DEV, copy.deepcopy(pc))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    assert torch.equal(a.arena.theta, b.arena.theta)


def test_results_do_not_depend_on_the_node_order():
    """The node order only changes which CTA row runs a node: a run with the node order reversed, launched eagerly,
    equals the captured run in the default order bit for bit."""
    from test_gpu_mnist import _problem
    outs = []
    for variant in ("default", "reversed"):
        pr = _problem(5, 32, "fused", XC, graph=nx.wheel_graph(5), M=100, eval_every=1000)
        pr.conf["input_pipeline"] = "resident"
        opt = CrossGradient(pr, DEV, copy.deepcopy(XC))
        prog = opt._program = RoundProgram(opt)
        if variant == "reversed":
            order = torch.arange(pr.placement.L - 1, -1, -1, dtype=torch.int32, device=DEV)
            prog.eng.t_node_order = order
            prog.eng._keep["node_order"] = order.data_ptr()
            prog.eng.op = type(prog.eng.op)(prog.eng._keep)
            prog.capturable = False
        opt.run_rounds(7)
        torch.cuda.synchronize()
        prog.eng.check()
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


def test_graph_replay_across_the_capture_boundary_equals_eager_launches():
    from test_gpu_mnist import _problem
    R = MAX_ROUNDS_PER_GRAPH + 6
    outs = []
    for capture in (False, True):
        conf = dict(XC, outer_iterations=R)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100, eval_every=1000)
        pr.conf["input_pipeline"] = "resident"
        opt = CrossGradient(pr, DEV, copy.deepcopy(conf))
        prog = opt._program = RoundProgram(opt)
        prog.capturable = capture
        assert prog.launches_per_round() == 4 + opt.dmax     # 3 + (1 + dmax)
        opt.run_rounds(R)
        torch.cuda.synchronize()
        assert bool(prog._graphs) == capture
        assert int(prog.eng.round_ctr.item()) == 2 * R
        prog.eng.check()
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(XC, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = CrossGradient(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), pr.forward_cnt, pr.calls.copy()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic():
    from test_gpu_mnist import _problem
    outs = []
    for _ in range(2):
        pr = _problem(5, 32, "fused", XC, graph=nx.wheel_graph(5), eval_every=3)
        opt = CrossGradient(pr, DEV, copy.deepcopy(XC))
        opt.train()
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(XC, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = CrossGradient(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = CrossGradient(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = CrossGradient(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes():
    """``debug_sequence_check``: every publication of both protocol rounds is tagged with its round; the fused run
    matches the PyTorch ops on the same fused forward/backward kernels."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(XC, debug_sequence_check=True, consensus_backend="auto" if backend == "fused" else "torch")
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        opt = CrossGradient(pr, DEV, copy.deepcopy(conf))
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            eng = opt._program.eng
            assert eng.seq_buf is not None
            torch.cuda.synchronize()
            err = int(eng.err.item())
            print(f"\nsequence check: err == {err}")
            assert err == 0
            eng.check()
    _assert_mostly_close(outs[0], outs[1])


def test_bytes_and_gradient_evaluations_per_round():
    from test_gpu_mnist import _problem
    pr = _problem(5, 32, "fused", XC, graph=nx.wheel_graph(5), M=100, eval_every=1000)
    opt = CrossGradient(pr, DEV, copy.deepcopy(XC))
    prog = opt._program = RoundProgram(opt)
    b, row = prog.eng.bytes_per_round(), pr.arena.n_pad * 4
    assert b["pulled_theta"] == b["pulled_cross"] == row * 16 and b["pulled"] == 2 * row * 16
    assert prog.eng.grad_evals() == {"useful": 5 + 16, "launched": 5 * 5}
