"""DSGD with momentum on the fused sm_90a kernels: ``dsgd_mix_kernel`` and ``dsgdm_step_kernel`` (local and
quasi-global momentum, Nesterov optional), one launch at a time against the float64 oracle with the bound of
``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err), then whole runs against the PyTorch path, determinism,
CUDA-graph replay and checkpoint/resume."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import dsgdm_oracle as mo
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, KernelProblem, _snap
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import DSGDm
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# every degree 0..9 appears: isolated (0..3), wheel5 (hub 4), star8 (hub 8), wheel10 (hub 9), random (5..7)
DM_GRAPHS = dict(GRAPHS, wheel5_ptr=[nx.wheel_graph(5)])
ROUNDS, CHECKED = 6, (0, 1, 5)
VARIANTS = [("local", False), ("local", True), ("quasi_global", False), ("quasi_global", True)]
VARIANT = pytest.mark.parametrize("momentum,nesterov", VARIANTS, ids=["local", "local-nest", "qg", "qg-nest"])
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:22s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, S, n, momentum, nesterov, n_pad=None, seed=0, mu=2.0, beta=0.9):
    conf = {"alg_name": "dsgdm", "alpha0": 0.08, "mu": mu, "beta": beta, "momentum": momentum, "nesterov": nesterov,
            "outer_iterations": ROUNDS, "profile": False}
    if graph_key.endswith("_ptr"):
        conf["complete_graph_mode"] = "pointer"
    pr = KernelProblem(DM_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    o = DSGDm(pr, DEV, conf)
    # the momentum rows hold garbage before round 0: the kernel must take them as zero there, not read them
    o.m[:, :n] = (1e3 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    if o.x_prev is not None:
        o.x_prev[:, :n] = (1e3 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    return pr, o, conf


def _state(pr, o, eng):
    s = _snap(pr, o, eng)
    t = lambda x: x.detach().double().cpu().numpy().copy()          # noqa: E731
    s["m"] = t(o.m)
    if o.x_prev is not None:
        s["x_prev"] = t(o.x_prev)
    return s


class Harness:
    def __init__(self, pr, o, conf):
        self.pr, self.o, self.conf = pr, o, conf
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.kind = conf["momentum"] + ("-nest" if conf["nesterov"] else "")
        want = co.dsgd_alpha_table(conf["alpha0"], conf["mu"], o.oits)
        self.alpha = self.eng.alpha.cpu().double().numpy()
        np.testing.assert_allclose(self.alpha, want, rtol=2 * self.u + 1e-14, atol=0)
        self.beta = float(NPDT[pr.dtype](conf["beta"]))
        self.n = max(s.offset + s.numel for s in pr.layout.slots)
        self.mhat_rows_equal = []

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        assert after["done_ctr"] == 0, name
        ends = name == "dsgdm_step"
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if ends else 0)), name
        for key in ("theta", "pub", "m", "x_prev"):
            if key in after:
                assert not after[key][..., self.n:].any(), f"{name}: padding of {key} written"
        if ends:
            assert np.array_equal(after["pub"][(k & 1) ^ 1, 0], after["theta"]), f"{name}: pub[par^1] != theta"
            if self.eng.sum_mode and self.o.quasi_global:
                self.mhat_rows_equal.append(bool((after["m"] == after["m"][0]).all()))
        if not check:
            return
        tp = Topology(self.pr.plan_graphs(self.o.oits, 0, 1)[k])
        if name == "local_sum":
            s, e = co.local_sum(before["pub"], k & 1)
            want, err = dict(before, sum_local=before["sum_local"].copy()), {"sum_local": np.zeros_like(before["sum_local"])}
            want["sum_local"][k & 1], err["sum_local"][k & 1] = s, e
        elif name == "dsgd_mix":
            sums = None
            if self.eng.sum_mode:
                s = before["sum_local"][k & 1]
                sums = (s, co.U64 * np.abs(s))
            want, err = co.dsgd_mix(before, k=k, nbrs=tp.neighbors_noself, W=tp.W, u=self.u,
                                    sum_mode=self.eng.sum_mode, sums=sums)
        else:
            want, err = mo.step(before, k=k, alpha=self.alpha[k], alpha_prev=self.alpha[k - 1] if k else 1.0,
                                beta=self.beta, quasi_global=self.o.quasi_global, nesterov=self.o.nesterov, u=self.u)
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name} round {k} {key}", got, want[key], err[key], C)
                kern = name if name != "dsgdm_step" else f"dsgdm_step {self.kind}"
                WORST[(kern, self.dt)] = max(WORST[(kern, self.dt)], r)
            else:
                assert np.array_equal(got, before[key]), f"{name} wrote {key}"

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            if self.eng.sum_mode:
                self.launch("local_sum", op.local_sum, k, check=chk)
            self.launch("dsgd_mix", op.dsgd_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("dsgdm_step", op.dsgdm_step, k, check=chk)
        self.eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@VARIANT
@pytest.mark.parametrize("graph_key", sorted(DM_GRAPHS))
def test_launches_match_oracle(graph_key, momentum, nesterov, dtype):
    """Every graph (degrees 0-9, complete graph in sum and pointer mode, a graph that changes every round), rows of 13
    parameters (padding in the row), S rotating with the case; round 0 starts from garbage momentum rows."""
    i = sorted(DM_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, momentum, nesterov, seed=i)
    h = Harness(pr, o, conf)
    assert h.eng.sum_mode == graph_key.endswith("_sum")
    h.run()


@DTYPES
@VARIANT
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, momentum, nesterov, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8 (degree-9 hub: both neighbor groups)."""
    pr, o, conf = _setup("wheel10", dtype, S, 77, momentum, nesterov, seed=S)
    Harness(pr, o, conf).run(rounds=3, checked=(0, 1, 2))


@DTYPES
@VARIANT
@pytest.mark.parametrize("size", ["one_vector", "grid_stride"])
def test_row_sizes_match_oracle(size, momentum, nesterov, dtype):
    """A row of exactly one vector, and rows long enough that the grid is capped at the resident CTAs and every
    thread walks the row more than once (the pre-wait loads only on the first iteration)."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, conf = _setup("random5to7", dtype, 5, vec, momentum, nesterov, n_pad=vec, seed=3)
        Harness(pr, o, conf).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, conf = _setup("random5to7", dtype, 17, 140001, momentum, nesterov, seed=4)
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o, conf).run(rounds=3, checked=(0, 1, 2))


@DTYPES
@pytest.mark.parametrize("nesterov", [False, True])
def test_sum_mode_mhat_rows_are_bitwise_equal_across_nodes(nesterov, dtype):
    """Complete graph through the network sum: every node's mixed row is the same S / N, so the quasi-global mhat rows
    are the same bits on every node after every round (also the garbage of round 0 is not read)."""
    pr, o, conf = _setup("complete6_sum", dtype, 3, 50, "quasi_global", nesterov, seed=9, mu=0.0)
    h = Harness(pr, o, conf)
    assert h.eng.sum_mode
    h.run(rounds=ROUNDS, checked=())
    assert h.mhat_rows_equal == [True] * ROUNDS
    m = o.m[:, :50]
    assert torch.equal(m, m[:1].expand_as(m)) and m.abs().max() > 0


@VARIANT
@pytest.mark.parametrize("graph_key", ["switch", "complete6_sum"])
def test_graph_replay_equals_eager_launches(graph_key, momentum, nesterov):
    """A captured RoundProgram gives, round after round, bitwise the state of the eager launches."""
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup(graph_key, torch.float32, 5, 300, momentum, nesterov, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            states.append(_state(pr, o, prog.eng))
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            if isinstance(x, np.ndarray):
                assert np.array_equal(x, b[key]), f"round {k}: {key}"
            else:
                assert x == b[key], f"round {k}: {key}"


# ------------------------------------------------------------------------------------------ whole runs ----
DM = {"alg_name": "dsgdm", "alpha0": 0.05, "mu": 0.01, "beta": 0.9, "momentum": "quasi_global", "nesterov": True,
      "outer_iterations": 7, "profile": False}
MODES = pytest.mark.parametrize("momentum", ["local", "quasi_global"])


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = DSGDm(a, DEV, copy.deepcopy(conf))
    ob = DSGDm(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


@MODES
def test_mnist_fp64_paper_shape_matches_torch_fp64(momentum):
    """The float64 conv-net kernel at the paper shape with the fp64 consensus kernels under CUDA graphs against autograd
    and the PyTorch ops in float64: within 1e-9 after one round and 1e-8 over the run."""
    from test_gpu_mnist import _generic_problem
    conf = dict(DM, momentum=momentum)
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine() and not ob._use_engine()
    oa.run_rounds(1)
    ob.run_rounds(1)
    torch.cuda.synchronize()
    assert _rel(a.arena.theta, b.arena.theta) < 1e-9
    oa.train()
    ob.train()
    assert _rel(a.arena.theta, b.arena.theta) < 1e-8
    assert _rel(oa.m, ob.m) < 1e-8
    assert a.forward_cnt == b.forward_cnt


@MODES
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete"])
def test_mnist_fp32_matches_torch_ops(graph, momentum):
    """fp32 tensor-core MNIST kernel, fused round programs against the PyTorch consensus ops driving the same fused
    forward/backward, with the tolerance of the other algorithms' fp32 comparison."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    N = 5
    G = {"cycle": nx.cycle_graph(N), "wheel": nx.wheel_graph(N), "complete": nx.complete_graph(N)}[graph]
    conf = dict(DM, momentum=momentum)
    a = _problem(N, 32, "fused", conf, graph=G, eval_every=3)
    b = _problem(N, 32, "fused", conf, graph=G, eval_every=3)
    oa, ob = _pair(a, b, conf)
    oa.train()
    ob.train()
    assert oa._program.eng.sum_mode == (graph == "complete")
    _assert_mostly_close(a.arena.theta, b.arena.theta)
    _assert_mostly_close(oa.m, ob.m)
    assert a.forward_cnt == b.forward_cnt
    assert len(a.metrics["validation_loss"]) == len(b.metrics["validation_loss"]) == 3


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    """Host-fed and staged rounds train exactly like the resident pipeline."""
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(DM, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = DSGDm(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.m.clone(), opt.x_prev.clone(), pr.forward_cnt, pr.calls.copy()))
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert torch.equal(x, y)
    assert outs[0][3] == outs[1][3] and (outs[0][4] == outs[1][4]).all()


@MODES
def test_density_fp64_matches_torch_fp64(momentum):
    from test_gpu_mlp_f64 import _density
    conf = dict(DM, momentum=momentum)
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine()
    oa.run_rounds(1)
    ob.run_rounds(1)
    torch.cuda.synchronize()
    assert _rel(a.arena.theta, b.arena.theta) < 1e-9
    oa.train()
    ob.train()
    assert _rel(a.arena.theta, b.arena.theta) < 1e-8
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


def test_density_fp32_matches_torch_ops():
    """fp32 density MLP on the tensor-core kernel: fused round programs against the PyTorch consensus ops driving the
    same fused forward/backward."""
    from test_gpu_mlp import _density_problem
    from test_gpu_mnist import _assert_mostly_close
    a = _density_problem("fused", B=500, M=1500, N=4)
    b = _density_problem("fused", B=500, M=1500, N=4)
    for pr in (a, b):
        pr.conf["optimizer_config"] = copy.deepcopy(DM)
    oa, ob = _pair(a, b, DM)
    oa.train()
    ob.train()
    assert oa._use_engine() and not ob._use_engine()
    _assert_mostly_close(a.arena.theta, b.arena.theta)
    assert a.forward_cnt == b.forward_cnt


def test_online_density_fp64_dynamic_graph_matches_torch_fp64(tmp_path):
    """The online problem (graph planned from the robot poses, changing over the run) in float64."""
    from test_gpu_mlp_f64 import _online_problem
    oc = dict(DM, alpha0=0.002, outer_iterations=9)
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    ref.arena.theta.copy_(fused.arena.theta)
    of = DSGDm(fused, DEV, copy.deepcopy(oc))
    DSGDm(ref, DEV, dict(copy.deepcopy(oc), consensus_backend="torch")).train()
    of.train()
    assert (fused.positions() == ref.positions()).all()
    assert fused.forward_cnt == ref.forward_cnt
    for key in ("validation_loss", "train_loss_moving_average"):
        torch.testing.assert_close(fused.metrics[key][-1], ref.metrics[key][-1], rtol=1e-9, atol=1e-12)
    assert _rel(fused.arena.theta, ref.arena.theta) < 1e-8


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", DM, graph=nx.wheel_graph(5), eval_every=3)
        opt = DSGDm(pr, DEV, copy.deepcopy(DM))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.m.clone(), opt.x_prev.clone()))
    for run in outs[1:]:
        for x, y in zip(run, outs[0]):
            assert torch.equal(x, y)


@MODES
@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model, momentum):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(DM, momentum=momentum, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = DSGDm(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = DSGDm(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = DSGDm(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.m, of.m)
    if momentum == "quasi_global":
        assert torch.equal(o2.x_prev, of.x_prev)
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_on_a_link_drop_run():
    """Link drops every round (several topology tables, isolated nodes) with ``debug_sequence_check``: no stale row is
    read, and the result matches the PyTorch ops walking the same graph sequence."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        pr = _problem(6, 32, "fused", DM, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 6}
        pr._init_faults()
        c = dict(copy.deepcopy(DM), debug_sequence_check=True,
                 consensus_backend="auto" if backend == "fused" else "torch")
        opt = DSGDm(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
