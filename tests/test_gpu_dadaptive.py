"""Decentralized AMSGrad / AdaGrad on the fused sm_90a kernels: ``dadaptive_mix_kernel`` (or ``dsgd_mix_kernel``) and
``dadaptive_step_kernel`` one launch at a time against the float64 oracle of ``tests/dadaptive_oracle.py`` with the
bound of ``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err), then whole runs against the PyTorch path, the
input pipelines, determinism, CUDA-graph replay, checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import dadaptive_oracle as do
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, KernelProblem, _snap
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import DAdaptive
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# every degree 0..9 appears: isolated (0..3), wheel5 (hub 4), star8 (hub 8), wheel10 (hub 9), random (5..7)
AD_GRAPHS = dict(GRAPHS, wheel5_ptr=[nx.wheel_graph(5)])
ROUNDS, CHECKED = 6, (0, 1, 5)
VARIANT = pytest.mark.parametrize("variant", ["amsgrad", "adagrad"])
TRACKING = pytest.mark.parametrize("tracking", [True, False], ids=["tracked", "own"])
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
ROWS = ("m", "v", "vhat", "ut")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:28s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _conf(variant, tracking, **kw):
    conf = dict({"alg_name": "dadaptive", "alpha": 0.01, "variant": variant, "tracking": tracking,
                 "outer_iterations": ROUNDS, "profile": False}, **kw)
    if variant == "amsgrad":
        conf.setdefault("beta2", 0.99)
    return conf


def _setup(graph_key, dtype, S, n, variant, tracking, n_pad=None, seed=0):
    conf = _conf(variant, tracking, beta1=0.8)
    if graph_key.endswith("_ptr"):
        conf["complete_graph_mode"] = "pointer"
    pr = KernelProblem(AD_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)

    def rnd(scale=1.0):
        return (scale * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)

    pr.arena.theta[:, :n] = rnd()
    o = DAdaptive(pr, DEV, conf)
    # a nonzero start (as after a resume): v above and below vhat so both sides of the max are taken, a tracker that
    # is not vhat, and some of it below eps so the clamp is taken too
    o.m[:, :n] = rnd(0.3)
    o.vhat[:, :n] = 1e-8 + rnd().abs()
    if o.v is not None:
        o.v[:, :n] = o.vhat[:, :n] * (0.5 + torch.rand(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV))
    if o.ut is not None:
        o.ut[:, :n] = o.vhat[:, :n] + rnd(0.3)
    return pr, o, conf


def _state(pr, o, eng):
    s = _snap(pr, o, eng)
    for name in ROWS:
        row = getattr(o, name)
        if row is not None:
            s[name] = row.detach().double().cpu().numpy().copy()
    return s


class Harness:
    def __init__(self, pr, o, conf):
        self.pr, self.o, self.conf = pr, o, conf
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        t = NPDT[pr.dtype]
        self.u = co.unit_roundoff(t)
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.alpha = self.eng.alpha.cpu().double().numpy()
        assert (self.alpha == float(t(conf["alpha"]))).all()
        # the constants as the kernel of this dtype holds them (representation, not round-off)
        self.beta1, self.beta2, self.eps = (float(t(x)) for x in (o.beta1, o.beta2, o.eps))
        self.n = max(s.offset + s.numel for s in pr.layout.slots)

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        assert after["done_ctr"] == 0, name
        step = name == "dadaptive_step"
        assert after["round_ctr"] == before["round_ctr"] + (1 if step else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if step else 0)), name
        for key in ("theta", "m", "v"):
            if key in after:
                assert not after[key][..., self.n:].any(), f"{name}: padding of {key} written"
        assert not after["pub"][:, 0, :, self.n:].any(), f"{name}: padding of the published theta written"
        if step:
            assert np.array_equal(after["pub"][(k & 1) ^ 1, 0], after["theta"]), f"{name}: pub[par^1] != theta"
        if not check:
            return
        tp = Topology(self.pr.plan_graphs(self.o.oits, 0, 1)[k])
        sums = None
        if self.eng.sum_mode:
            s = before["sum_local"][k & 1]
            sums = (s, co.U64 * np.abs(s))
        if name == "local_sum":
            s, e = co.local_sum(before["pub"], k & 1)
            want, err = dict(before, sum_local=before["sum_local"].copy()), {"sum_local": np.zeros_like(before["sum_local"])}
            want["sum_local"][k & 1], err["sum_local"][k & 1] = s, e
        elif name == "dsgd_mix":
            want, err = co.dsgd_mix(before, k=k, nbrs=tp.neighbors_noself, W=tp.W, u=self.u,
                                    sum_mode=self.eng.sum_mode, sums=sums)
        elif name == "dadaptive_mix":
            want, err = do.mix(before, k=k, nbrs=tp.neighbors_noself, W=tp.W, u=self.u,
                               sum_mode=self.eng.sum_mode, sums=sums)
        else:
            want, err = do.step(before, k=k, alpha=self.alpha[k], beta1=self.beta1, beta2=self.beta2, eps=self.eps,
                                variant=self.o.variant, tracking=self.o.tracking, u=self.u)
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name} round {k} {key}", got, want[key], err[key], C)
                kern = name if not step else f"dadaptive_step {self.o.variant} {'tr' if self.o.tracking else 'own'}"
                WORST[(kern, self.dt)] = max(WORST[(kern, self.dt)], r)
            else:
                assert np.array_equal(got, before[key]), f"{name} round {k} wrote {key}"

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            if self.eng.sum_mode:
                self.launch("local_sum", op.local_sum, k, check=chk)
            if self.o.tracking:
                self.launch("dadaptive_mix", op.dadaptive_mix, k, check=chk)
            else:
                self.launch("dsgd_mix", op.dsgd_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("dadaptive_step", op.dadaptive_step, k, check=chk)
        self.eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@VARIANT
@TRACKING
@pytest.mark.parametrize("graph_key", sorted(AD_GRAPHS))
def test_launches_match_oracle(graph_key, tracking, variant, dtype):
    """Every graph (degrees 0-9, the complete graph in sum and pointer mode, a graph that changes every round), rows of
    13 parameters (padding in the row), S rotating with the case."""
    i = sorted(AD_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, variant, tracking, seed=i)
    h = Harness(pr, o, conf)
    assert h.eng.sum_mode == graph_key.endswith("_sum")
    assert h.eng.C == (2 if tracking else 1)
    h.run()


@DTYPES
@VARIANT
@TRACKING
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, tracking, variant, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8 (degree-9 hub: both neighbor pair groups)."""
    pr, o, conf = _setup("wheel10", dtype, S, 77, variant, tracking, seed=S)
    Harness(pr, o, conf).run(rounds=3, checked=(0, 1, 2))


@DTYPES
@VARIANT
@TRACKING
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, tracking, variant, dtype):
    """A row of exactly one vector, a row padded well past its parameters, and rows long enough that the grid is capped
    at the resident CTAs and every thread walks the row more than once (the pre-wait loads on every iteration)."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, conf = _setup("random5to7", dtype, 5, vec, variant, tracking, n_pad=vec, seed=3)
        Harness(pr, o, conf).run()
        return
    if size == "padded":
        pr, o, conf = _setup("cycle6", dtype, 3, 9, variant, tracking, n_pad=64 * vec, seed=5)
        Harness(pr, o, conf).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, conf = _setup("random5to7", dtype, 17, 140001, variant, tracking, seed=4)
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@VARIANT
@TRACKING
@pytest.mark.parametrize("graph_key", ["switch", "complete6_sum"])
def test_graph_replay_equals_eager_launches(graph_key, tracking, variant):
    """A captured RoundProgram gives, round after round, bitwise the state of the eager launches."""
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup(graph_key, torch.float32, 5, 300, variant, tracking, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        assert prog.launches_per_round() == (1 if prog.eng.sum_mode else 0) + 3
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
AD = {"alg_name": "dadaptive", "alpha": 0.002, "variant": "amsgrad", "tracking": True, "outer_iterations": 7,
      "profile": False}
CASES = pytest.mark.parametrize("variant,tracking", [("amsgrad", True), ("adagrad", True), ("amsgrad", False),
                                                     ("adagrad", False)],
                                ids=["amsgrad-tracked", "adagrad-tracked", "amsgrad-own", "adagrad-own"])


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = DAdaptive(a, DEV, copy.deepcopy(conf))
    ob = DAdaptive(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


def _rows_close(oa, ob, bound):
    if getattr(oa, "_program", None) is not None:
        oa._program.sync_back()
    for name in oa.STATE:
        r = _rel(getattr(oa, name), getattr(ob, name))
        assert r < bound, f"{name}: {r:.2e}"


@CASES
def test_mnist_fp64_paper_shape_matches_torch_fp64(variant, tracking):
    """The float64 conv-net kernel at the paper shape with the fp64 consensus kernels under CUDA graphs against autograd
    and the PyTorch ops in float64, within the 1e-8 whole-run bound of the other algorithms."""
    from test_gpu_mnist import _generic_problem
    conf = dict(AD, variant=variant, tracking=tracking)
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine() and not ob._use_engine()
    oa.run_rounds(1)
    ob.run_rounds(1)
    torch.cuda.synchronize()
    r1 = _rel(a.arena.theta, b.arena.theta)
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64 {variant} tracking={tracking}: rel after 1 round {r1:.2e}, after the run {r:.2e}")
    assert r1 < 1e-9 and r < 1e-8
    _rows_close(oa, ob, 1e-8)
    assert a.forward_cnt == b.forward_cnt


@CASES
def test_density_fp64_matches_torch_fp64(variant, tracking):
    from test_gpu_mlp_f64 import _density
    conf = dict(AD, variant=variant, tracking=tracking)
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64 {variant} tracking={tracking}: rel {r:.2e}")
    assert r < 1e-8
    _rows_close(oa, ob, 1e-8)
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


@VARIANT
def test_online_density_fp64_dynamic_graph_matches_torch_fp64(tmp_path, variant):
    """The online problem (graph planned from the robot poses, changing over the run) in float64, tracked."""
    from test_gpu_mlp_f64 import _online_problem
    oc = dict(AD, variant=variant, alpha=0.0005, outer_iterations=9)
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    ref.arena.theta.copy_(fused.arena.theta)
    of = DAdaptive(fused, DEV, copy.deepcopy(oc))
    orf = DAdaptive(ref, DEV, dict(copy.deepcopy(oc), consensus_backend="torch"))
    orf.train()
    of.train()
    assert len(of._program.eng.topos) > 1
    assert (fused.positions() == ref.positions()).all()
    assert fused.forward_cnt == ref.forward_cnt
    for key in ("validation_loss", "train_loss_moving_average"):
        torch.testing.assert_close(fused.metrics[key][-1], ref.metrics[key][-1], rtol=1e-9, atol=1e-12)
    r = _rel(fused.arena.theta, ref.arena.theta)
    print(f"\nonline density fp64 {variant}: rel {r:.2e}")
    assert r < 1e-8
    _rows_close(of, orf, 1e-8)


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    """Host-fed and staged rounds train exactly like the resident pipeline."""
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(AD, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = DAdaptive(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.m.clone(), opt.v.clone(), opt.vhat.clone(), opt.ut.clone(),
                     pr.forward_cnt, pr.calls.copy()))
    for x, y in zip(outs[0][:5], outs[1][:5]):
        assert torch.equal(x, y)
    assert outs[0][5] == outs[1][5] and (outs[0][6] == outs[1][6]).all()


# ------------------------------------------------------------------------- determinism and resume ----
@VARIANT
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch, variant):
    from test_gpu_mnist import _problem
    conf = dict(AD, variant=variant)
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = DAdaptive(pr, DEV, copy.deepcopy(conf))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append([pr.arena.theta.clone()] + [getattr(opt, n).clone() for n in opt.STATE])
    for run in outs[1:]:
        for x, y in zip(run, outs[0]):
            assert torch.equal(x, y)


@CASES
@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model, variant, tracking):
    """Resume at round 3: the published tracker comes back from the checkpoint and AdaGrad's count from the round
    counter."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(AD, variant=variant, tracking=tracking, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = DAdaptive(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = DAdaptive(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = DAdaptive(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in o2.STATE:
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt


@VARIANT
@TRACKING
def test_sequence_check_passes_on_a_link_drop_run(variant, tracking):
    """Link drops every round (several topology tables, isolated nodes) with ``debug_sequence_check``: no stale row is
    read, and the result matches the PyTorch ops walking the same graph sequence."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(AD, variant=variant, tracking=tracking)
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 7}
        pr._init_faults()
        c = dict(copy.deepcopy(conf), debug_sequence_check=True,
                 consensus_backend="auto" if backend == "fused" else "torch")
        opt = DAdaptive(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
