"""GT-HSGD on the fused sm_90a kernels: ``hsgd_track_kernel`` one launch at a time against the float64 oracle with the
bound of ``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err); the prev-point forward/backward of every
training kernel on the same minibatch (bit for bit at theta_prev = theta, against float64 autograd elsewhere) in the
resident, staged and host pipelines; the draw counters; whole runs against the PyTorch path and against fused DSGT;
CUDA-graph replay across the 64-round capture boundary; pipelines, determinism, checkpoint/resume and the sequence
check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import hsgd_oracle as ho
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, GradSource, KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import MAX_ROUNDS_PER_GRAPH, RoundProgram
from nn_distributed_training_b200.optimizers import DSGT, GTHSGD
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# degrees 0..16: isolated (0..3), path2 (1), cycle6 (2), random (5..7), complete6 in sum and pointer mode (5),
# star8 (hub 8), wheel10 (hub 9), star16 (hub 16), and a graph that changes every round
HS_GRAPHS = dict(GRAPHS)
HS_GRAPHS["star16"] = [nx.star_graph(16)]
ROUNDS = 4
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per output and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:22s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
class PairSource(GradSource):
    """GradSource with a second, prev-point set of partials (other seeded values, the same draw counter)."""

    def __init__(self, L, S, n, n_pad, dtype, seed):
        super().__init__(L, S, n, n_pad, dtype, seed)
        self.prev = GradSource(L, S, n, n_pad, dtype, seed + 1000)
        self.grad_part_prev = self.prev.grad_part

    def enable_prev_point(self, theta_prev):
        pass

    def launch_prev(self):
        self.prev.calls.copy_(self.calls)
        self.prev.launch()


class PairProblem(KernelProblem):
    def __init__(self, graphs, n, dtype, S, seed=0, n_pad=None, conf=None):
        super().__init__(graphs, n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
        self.fused = PairSource(self.N, S, n, self.layout.n_pad, dtype, seed)
        self.fused.pr_calls = self.calls


def _setup(graph_key, dtype, S, n, beta, n_pad=None, seed=0, mode="sum"):
    conf = {"alg_name": "gt_hsgd", "alpha": 0.08, "beta": beta, "outer_iterations": ROUNDS, "profile": False,
            "complete_graph_mode": mode}
    pr = PairProblem(HS_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    rnd = lambda: torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)  # noqa: E731
    pr.arena.theta[:, :n] = rnd()
    o = GTHSGD(pr, DEV, conf)
    # a nonzero start (as after a resume) exercises every term, also round 0's v (read for v' - v, not for v')
    o.y[:, :n] = rnd()
    o.v[:, :n] = rnd()
    o.theta_prev[:, :n] = rnd()
    return pr, o


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def run_checked(pr, o, rounds=ROUNDS):
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    u = co.unit_roundoff(NPDT[pr.dtype])
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    n = pr.n
    src, op = pr.fused, eng.op
    for k in range(rounds):
        if eng.sum_mode:
            op.local_sum()
        op.dsgt_mix()
        src.launch()
        src.launch_prev()
        torch.cuda.synchronize()
        par = k & 1
        pub0, th, v0 = _t(eng.pub), _t(pr.arena.theta), _t(o.v)
        gpart, gppart, calls0 = _t(src.grad_part), _t(src.grad_part_prev), src.calls.cpu().numpy().copy()
        op.hsgd_track()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == k + 1 and int(eng.done_ctr.item()) == 0
        assert np.array_equal(src.calls.cpu().numpy(), calls0 + 1)
        pub1, v1, tp1 = _t(eng.pub), _t(o.v), _t(o.theta_prev)
        assert np.array_equal(tp1, th) and np.array_equal(pub1[par ^ 1, 0, :pr.N], th)
        assert np.array_equal(pub1[par], pub0[par]), "the round's own parity was written"
        for key, arr in (("pub", pub1), ("v", v1), ("theta_prev", tp1)):
            assert not arr[..., n:].any(), f"padding of {key} written"
        tp = Topology(pr.plan_graphs(o.oits, 0, 1)[k])
        for l in range(pr.N):
            nb = tp.neighbors_noself[l]
            if eng.sum_mode:     # y = S_y / N: every node a neighbor with weight 1 / N
                w_self, w_nbr, nb = 1.0 / pr.N, [1.0 / pr.N] * (pr.N - 1), [j for j in range(pr.N) if j != l]
            else:
                w_self, w_nbr = tp.W[l, l], [tp.W[l, j] for j in nb]
            (yn, vn), (ey, ev) = ho.hsgd_track(pub0[par, 1, l, :n], w_self, w_nbr, [pub0[par, 1, j, :n] for j in nb],
                                               gpart[l, :, :n], gppart[l, :, :n], v0[l, :n], th[l, :n], o.omb,
                                               k == 0, u)
            r = co.check(f"round {k} node {l} y", pub1[par ^ 1, 1, l, :n], yn, ey, C)
            WORST[("y", dt)] = max(WORST[("y", dt)], r)
            r = co.check(f"round {k} node {l} v", v1[l, :n], vn, ev, C)
            WORST[("v", dt)] = max(WORST[("v", dt)], r)
    eng.check()
    return eng


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(HS_GRAPHS))
def test_launches_match_oracle(graph_key, dtype):
    """Every graph (degrees 0-16, the complete graph in sum and pointer mode, a changing graph), rows of 13 parameters
    (padding in the row), round 0 and later rounds, S and beta rotating with the case."""
    i = sorted(HS_GRAPHS).index(graph_key)
    mode = "pointer" if graph_key.endswith("_ptr") else "sum"
    pr, o = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, (1.0, 0.5, 0.1, 0.01)[i % 4], seed=i, mode=mode)
    eng = run_checked(pr, o)
    assert eng.C == 2 and eng.sum_mode == (graph_key == "complete6_sum")


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The 4-deep and 8-deep partial sums of both sets and the tail loop past 8 (degree-16 hub)."""
    pr, o = _setup("star16", dtype, S, 77, 0.3, seed=S)
    run_checked(pr, o, rounds=2)


@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    """A row of exactly one vector, a padded row, and rows long enough that the grid is capped at the resident CTAs and
    every thread walks the row more than once."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o = _setup("random5to7", dtype, 5, vec, 0.2, n_pad=vec, seed=3)
    elif size == "padded":
        pr, o = _setup("random5to7", dtype, 3, 3 * vec + 1, 0.2, seed=5)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o = _setup("random5to7", dtype, 17, 140001, 0.2, seed=4)
        assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    run_checked(pr, o, rounds=2)


# ------------------------------------------------------------------------- prev-point forward/backward ----
HC = {"alg_name": "gt_hsgd", "alpha": 0.01, "beta": 0.3, "outer_iterations": 7, "profile": False}


def _mnist(kind, backend="fused", conf=None):
    from test_gpu_mnist import _generic_problem, _problem
    conf = copy.deepcopy(conf or HC)
    if kind == "fp64_cluster":
        return _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=5, conf=conf)
    if kind == "fp32_cluster":
        return _problem(4, 32, backend, conf, M=100)
    if kind == "batch_split":
        return _problem(4, 96, backend, conf, M=200)
    return _generic_problem((4, 3, 32), torch.float32, backend, B=32, N=4, conf=conf)      # generic conv net


def _mlp(kind, tmp):
    if kind == "mlp_bf16":
        from test_gpu_mlp import _density_problem
        return _density_problem("fused", B=500, M=1500, N=4)
    if kind == "mlp_fp64":
        from test_gpu_mlp_f64 import _density
        return _density(4, 500, M=700, opt_conf=copy.deepcopy(HC))
    from test_gpu_mlp import _online_problem
    return _online_problem("fused", tmp, copy.deepcopy(HC))


KERNELS = ["fp64_cluster", "fp32_cluster", "batch_split", "generic", "mlp_bf16", "mlp_fp64", "online_density"]


@pytest.mark.parametrize("kind", KERNELS)
def test_prev_point_at_theta_equals_the_current_point_bit_for_bit(kind, tmp_path):
    """theta_prev = theta: both launches draw the same minibatch and compute the same partials, bit for bit, twice in a
    row (the draw counters of both ops advance together)."""
    pr = _mnist(kind) if kind in KERNELS[:4] else _mlp(kind, str(tmp_path))
    fz = pr.fused
    o = GTHSGD(pr, DEV, copy.deepcopy(HC))
    assert fz.prev_op is not None
    o.theta_prev.copy_(pr.arena.theta)
    # the bf16 MLP kernel (float32 arena, csrc/mlp_tc.cu) adds the output layer's w4 and b4 gradients with shared-memory
    # float atomics, so those two slots vary in their last bits from launch to launch of the same op: bit for bit up to
    # them, to float32 summation order on them
    atomics = kind in ("mlp_bf16", "online_density")
    cut = pr.layout.slots[-2].offset if atomics else pr.arena.n_pad
    for _ in range(2):
        fz.launch()
        fz.launch_prev()
        torch.cuda.synchronize()
        assert torch.equal(fz.grad_part[..., :cut], fz.grad_part_prev[..., :cut])
        if atomics:
            torch.testing.assert_close(fz.grad_part, fz.grad_part_prev, rtol=1e-5, atol=1e-7)
        assert fz.grad_part.abs().sum() > 0
        if hasattr(fz, "calls_prev"):
            assert torch.equal(fz.calls, fz.calls_prev)
        else:
            fz.calls += 1           # the consensus step's bookkeeping
    print(f"\n{kind}: {getattr(fz, 'kernel_name', type(fz).__name__)}")


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_prev_point_direct_ops_read_the_staged_batch(pipeline):
    """The staged and host pipelines: the prev-point direct op reads the stage slot of step 0, so at theta_prev = theta
    it gives the direct training op's partials bit for bit, in both stage sets."""
    pr = _mnist("fp32_cluster")
    pr.conf["input_pipeline"] = pipeline
    o = GTHSGD(pr, DEV, copy.deepcopy(HC))
    prog = o._program = RoundProgram(o)
    assert prog.pipeline == pipeline and prog.launches_per_round() == 5
    fz = pr.fused
    o.theta_prev.copy_(pr.arena.theta)
    for b in (0, 1):
        fz.gather_ops[b].launch()
        fz.direct_ops[b][0].train()
        fz.direct_prev_ops[b].train()
        torch.cuda.synchronize()
        assert torch.equal(fz.grad_part, fz.grad_part_prev), b
        assert torch.equal(fz.calls, fz.calls_prev)


def test_prev_point_gradient_matches_fp64_autograd_on_the_sampler_batch():
    """theta_prev != theta: the float64 cluster kernel's prev-point gradient against autograd at theta_prev on the
    batch the sampler draws (the autograd path of compute_grads_pair)."""
    a = _mnist("fp64_cluster")
    b = _mnist("fp64_cluster", backend="torch")
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = GTHSGD(a, DEV, copy.deepcopy(HC)), GTHSGD(b, DEV, dict(copy.deepcopy(HC), consensus_backend="torch"))
    g = torch.Generator().manual_seed(3)
    tp = (a.arena.theta.cpu() + 0.05 * torch.randn(a.arena.theta.shape, generator=g, dtype=torch.float64)).to(DEV)
    tp[:, a.n:] = 0
    oa.theta_prev.copy_(tp)
    ob.theta_prev.copy_(tp)
    ga, gb = a.arena.zeros(), b.arena.zeros()
    a.compute_grads_pair(oa.theta_prev, ga)
    b.compute_grads_pair(ob.theta_prev, gb)
    torch.cuda.synchronize()
    for got, want in ((a.arena.grad, b.arena.grad), (ga, gb)):
        r = ((got - want).norm() / want.norm()).item()
        print(f"\nfp64 cluster vs autograd: rel {r:.2e}")
        assert r < 1e-12
    assert (a.calls == b.calls).all() and a.forward_cnt == b.forward_cnt


@pytest.mark.parametrize("pipeline", ["resident", "staged", "host"])
def test_draw_counters_of_both_ops_equal_the_host_mirror(pipeline):
    pr = _mnist("fp32_cluster", conf=dict(HC, outer_iterations=12))
    pr.conf["input_pipeline"] = pipeline
    o = GTHSGD(pr, DEV, dict(HC, outer_iterations=12))
    o.run_rounds(5)
    o.run_rounds(4)
    torch.cuda.synchronize()
    want = torch.as_tensor(pr.calls.astype(np.int32), device=DEV)
    assert (pr.calls == 9).all()
    assert torch.equal(pr.fused.calls, want) and torch.equal(pr.fused.calls_prev, want)


# ------------------------------------------------------------------------------------------ whole runs ----
def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = GTHSGD(a, DEV, copy.deepcopy(conf))
    ob = GTHSGD(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


def test_mnist_fp64_paper_shape_matches_torch_fp64():
    """The float64 conv-net kernels (both points) at the paper shape with the fp64 consensus kernels under CUDA graphs
    against autograd and the PyTorch ops in float64."""
    from test_gpu_mnist import _generic_problem
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(HC))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(HC))
    oa, ob = _pair(a, b, HC)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64: rel {r:.2e}, y {_rel(oa.y, ob.y):.2e}, v {_rel(oa.v, ob.v):.2e}")
    assert r < 1e-10
    for name in ("y", "v", "theta_prev"):
        assert _rel(getattr(oa, name), getattr(ob, name)) < 1e-10, name
    assert a.forward_cnt == b.forward_cnt


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(HC))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(HC))
    oa, ob = _pair(a, b, HC)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64: rel {r:.2e}, y {_rel(oa.y, ob.y):.2e}, v {_rel(oa.v, ob.v):.2e}")
    assert r < 1e-10
    assert _rel(oa.y, ob.y) < 1e-10 and _rel(oa.v, ob.v) < 1e-10
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_beta_one_is_fused_dsgt_bit_for_bit(model):
    """beta = 1 on the fused kernels equals fused DSGT with init_grads false, bit for bit."""
    conf = dict(HC, beta=1.0, outer_iterations=12)
    dconf = {"alg_name": "dsgt", "alpha": HC["alpha"], "init_grads": False, "outer_iterations": 12, "profile": False}
    if model == "mnist_fp32":
        a, b = _mnist("fp32_cluster", conf=conf), _mnist("fp32_cluster", conf=dconf)
    else:
        from test_gpu_mlp_f64 import _density
        a, b = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf)), _density(4, 500, M=700, opt_conf=copy.deepcopy(dconf))
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = GTHSGD(a, DEV, copy.deepcopy(conf)), DSGT(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    assert torch.equal(a.arena.theta, b.arena.theta)
    assert torch.equal(oa.y, ob.y) and torch.equal(oa.v, ob.g)


def test_graph_replay_across_the_capture_boundary_equals_eager_launches():
    from test_gpu_mnist import _problem
    R = MAX_ROUNDS_PER_GRAPH + 6
    outs = []
    for capture in (False, True):
        conf = dict(HC, outer_iterations=R)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100, eval_every=1000)
        pr.conf["input_pipeline"] = "resident"
        opt = GTHSGD(pr, DEV, copy.deepcopy(conf))
        prog = opt._program = RoundProgram(opt)
        prog.capturable = capture
        assert prog.launches_per_round() == 4
        opt.run_rounds(R)
        torch.cuda.synchronize()
        assert bool(prog._graphs) == capture
        assert int(prog.eng.round_ctr.item()) == R
        prog.eng.check()
        prog.sync_back()
        outs.append((pr.arena.theta.clone(), opt.y.clone(), opt.v.clone(), opt.theta_prev.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(HC, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = GTHSGD(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.y.clone(), opt.v.clone(), opt.theta_prev.clone(), pr.forward_cnt,
                     pr.calls.copy()))
    for x, y in zip(outs[0][:4], outs[1][:4]):
        assert torch.equal(x, y)
    assert outs[0][4] == outs[1][4] and (outs[0][5] == outs[1][5]).all()


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic():
    from test_gpu_mnist import _problem
    outs = []
    for _ in range(2):
        pr = _problem(5, 32, "fused", HC, graph=nx.wheel_graph(5), eval_every=3)
        opt = GTHSGD(pr, DEV, copy.deepcopy(HC))
        opt.train()
        outs.append((pr.arena.theta.clone(), opt.y.clone(), opt.v.clone(), opt.theta_prev.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(HC, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = GTHSGD(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = GTHSGD(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = GTHSGD(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in ("y", "v", "theta_prev"):
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes():
    """``debug_sequence_check``: every hsgd_track publication is tagged with its round; the fused run matches the
    PyTorch ops on the same fused forward/backward kernels."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(HC, debug_sequence_check=True, consensus_backend="auto" if backend == "fused" else "torch")
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        opt = GTHSGD(pr, DEV, copy.deepcopy(conf))
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
