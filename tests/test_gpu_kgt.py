"""K-GT and local DSGD on the fused sm_90a kernels: ``kgt_mix_kernel`` (or ``dsgd_mix_kernel``) and
``kgt_step_kernel`` at every step index, one launch at a time against the float64 oracle with the bound of
``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err), then whole runs against the PyTorch path and against
fused DSGT / DSGD, the input pipelines, determinism, CUDA-graph replay, checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import kgt_oracle as ko
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, KernelProblem, _snap
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import DSGD, DSGT, KGT
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# every degree 0..9 appears: isolated (0..3), wheel5 (hub 4), star8 (hub 8), wheel10 (hub 9), random (5..7)
KG_GRAPHS = dict(GRAPHS, wheel5_ptr=[nx.wheel_graph(5)])
ROUNDS, CHECKED = 6, (0, 1, 5)
CORR = pytest.mark.parametrize("correction", [True, False], ids=["kgt", "local_dsgd"])
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:22s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, S, n, K, correction, n_pad=None, seed=0):
    conf = {"alg_name": "kgt", "alpha": 0.08, "local_steps": K, "correction": correction,
            "outer_iterations": ROUNDS, "profile": False}
    if graph_key.endswith("_ptr"):
        conf["complete_graph_mode"] = "pointer"
    pr = KernelProblem(KG_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    o = KGT(pr, DEV, conf)
    if correction:
        # a nonzero start (as after a resume) exercises every term of the mix; d holds garbage before step 0, which
        # the kernel must not read
        o.c[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        o.y[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        o.d[:, :n] = (1e3 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    return pr, o, conf


def _state(pr, o, eng):
    s = _snap(pr, o, eng)
    t = lambda x: x.detach().double().cpu().numpy().copy()          # noqa: E731
    if o.correction:
        s["c"] = t(o.c)
        s["d"] = t(o.d)
    return s


class Harness:
    def __init__(self, pr, o, conf):
        self.pr, self.o, self.conf = pr, o, conf
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, o.local_steps))
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.alpha = self.eng.alpha.cpu().double().numpy()
        assert (self.alpha == float(NPDT[pr.dtype](conf["alpha"]))).all()
        self.n = max(s.offset + s.numel for s in pr.layout.slots)
        self.K = o.local_steps

    def launch(self, name, fn, k, p=0, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        assert after["done_ctr"] == 0, name
        step = name == "kgt_step"
        ends = step and p == self.K - 1
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if step else 0)), name
        for key in ("theta", "pub", "c", "d"):
            if key in after:
                assert not after[key][..., self.n:].any(), f"{name}: padding of {key} written"
        if ends:
            assert np.array_equal(after["pub"][(k & 1) ^ 1, 0], after["theta"]), f"{name}: pub[par^1] != theta"
        if not check:
            return
        tp = Topology(self.pr.plan_graphs(self.o.oits, 0, self.K)[k])
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
        elif name == "kgt_mix":
            want, err = ko.mix(before, k=k, nbrs=tp.neighbors_noself, W=tp.W, u=self.u,
                               sum_mode=self.eng.sum_mode, sums=sums)
        else:
            want, err = ko.step(before, k=k, p=p, K=self.K, alpha=self.alpha[k], correction=self.o.correction, u=self.u)
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name}({p}) round {k} {key}", got, want[key], err[key], C)
                kern = name if name != "kgt_step" else f"kgt_step {'corr' if self.o.correction else 'local'}"
                WORST[(kern, self.dt)] = max(WORST[(kern, self.dt)], r)
            elif name == "kgt_step" and key == "d" and p == self.K - 1:
                continue                  # d is dead after the last step (not stored, not compared)
            else:
                assert np.array_equal(got, before[key]), f"{name}({p}) wrote {key}"

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            if self.eng.sum_mode:
                self.launch("local_sum", op.local_sum, k, check=chk)
            if self.o.correction:
                self.launch("kgt_mix", op.kgt_mix, k, check=chk)
            else:
                self.launch("dsgd_mix", op.dsgd_mix, k, check=chk)
            for p in range(self.K):
                self.launch("grad", src.launch, k)
                self.launch("kgt_step", lambda: op.kgt_step(p), k, p=p, check=chk)
        self.eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@CORR
@pytest.mark.parametrize("graph_key", sorted(KG_GRAPHS))
def test_launches_match_oracle(graph_key, correction, dtype):
    """Every graph (degrees 0-9, complete graph in sum and pointer mode, a graph that changes every round), rows of 13
    parameters (padding in the row), S and K rotating with the case; d holds garbage before step 0."""
    i = sorted(KG_GRAPHS).index(graph_key)
    K = (1, 2, 3)[i % 3]
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, K, correction, seed=i)
    h = Harness(pr, o, conf)
    assert h.eng.sum_mode == graph_key.endswith("_sum")
    assert h.eng.C == (2 if correction else 1)
    h.run()


@DTYPES
@CORR
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, correction, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8 (degree-9 hub: both neighbor pairs groups)."""
    pr, o, conf = _setup("wheel10", dtype, S, 77, 3, correction, seed=S)
    Harness(pr, o, conf).run(rounds=3, checked=(0, 1, 2))


@DTYPES
@CORR
@pytest.mark.parametrize("size", ["one_vector", "grid_stride"])
def test_row_sizes_match_oracle(size, correction, dtype):
    """A row of exactly one vector, and rows long enough that the grid is capped at the resident CTAs and every
    thread walks the row more than once (the pre-wait loads only on the first iteration)."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, conf = _setup("random5to7", dtype, 5, vec, 2, correction, n_pad=vec, seed=3)
        Harness(pr, o, conf).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, conf = _setup("random5to7", dtype, 17, 140001, 2, correction, seed=4)
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@CORR
@pytest.mark.parametrize("graph_key", ["switch", "complete6_sum"])
def test_graph_replay_equals_eager_launches(graph_key, correction):
    """A captured RoundProgram gives, round after round, bitwise the state of the eager launches."""
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup(graph_key, torch.float32, 5, 300, 3, correction, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        assert prog.launches_per_round() == (1 if prog.eng.sum_mode else 0) + 1 + 2 * 3
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            st = _state(pr, o, prog.eng)
            st.pop("d", None)
            states.append(st)
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            if isinstance(x, np.ndarray):
                assert np.array_equal(x, b[key]), f"round {k}: {key}"
            else:
                assert x == b[key], f"round {k}: {key}"


# ------------------------------------------------------------------------------------------ whole runs ----
KG = {"alg_name": "kgt", "alpha": 0.01, "local_steps": 2, "correction": True, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = KGT(a, DEV, copy.deepcopy(conf))
    ob = KGT(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


@CORR
def test_mnist_fp64_paper_shape_matches_torch_fp64(correction):
    """The float64 conv-net kernel at the paper shape with the fp64 consensus kernels under CUDA graphs against autograd
    and the PyTorch ops in float64, within the 1e-8 whole-run bound of the other algorithms."""
    from test_gpu_mnist import _generic_problem
    conf = dict(KG, correction=correction)
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
    print(f"\nMNIST fp64 correction={correction}: rel after 1 round {r1:.2e}, after the run {r:.2e}")
    assert r1 < 1e-9 and r < 1e-8
    if correction:
        assert _rel(oa.c, ob.c) < 1e-8 and _rel(oa.y, ob.y) < 1e-8
    assert a.forward_cnt == b.forward_cnt


@CORR
def test_density_fp64_matches_torch_fp64(correction):
    from test_gpu_mlp_f64 import _density
    conf = dict(KG, correction=correction)
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64 correction={correction}: rel {r:.2e}")
    assert r < 1e-8
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


def test_online_density_fp64_dynamic_graph_matches_torch_fp64(tmp_path):
    """The online problem (graph planned from the robot poses, changing over the run; K = 2 draws per round) in
    float64."""
    from test_gpu_mlp_f64 import _online_problem
    oc = dict(KG, alpha=0.002, outer_iterations=9)
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    ref.arena.theta.copy_(fused.arena.theta)
    of = KGT(fused, DEV, copy.deepcopy(oc))
    KGT(ref, DEV, dict(copy.deepcopy(oc), consensus_backend="torch")).train()
    of.train()
    assert len(of._program.eng.topos) > 1
    assert (fused.positions() == ref.positions()).all()
    assert fused.forward_cnt == ref.forward_cnt
    for key in ("validation_loss", "train_loss_moving_average"):
        torch.testing.assert_close(fused.metrics[key][-1], ref.metrics[key][-1], rtol=1e-9, atol=1e-12)
    r = _rel(fused.arena.theta, ref.arena.theta)
    print(f"\nonline density fp64: rel {r:.2e}")
    assert r < 1e-8


def test_fused_one_local_step_is_fused_dsgt():
    """K = 1 on the fused kernels: the mixed row theta + alpha y and the tracker equal fused DSGT's (init_grads
    false) to rounding."""
    from test_gpu_mlp_f64 import _density
    alpha = 0.01
    conf = dict(KG, alpha=alpha, local_steps=1, outer_iterations=12)
    dconf = {"alg_name": "dsgt", "alpha": alpha, "init_grads": False, "outer_iterations": 12, "profile": False}
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, opt_conf=copy.deepcopy(dconf))
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = KGT(a, DEV, copy.deepcopy(conf)), DSGT(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    x = a.arena.theta + alpha * oa.y
    rx, ry = _rel(x, b.arena.theta), _rel(oa.y, ob.y)
    print(f"\nfused K-GT K=1 vs fused DSGT: mixed rows {rx:.2e}, trackers {ry:.2e}")
    assert rx < 1e-10 and ry < 1e-10


@pytest.mark.parametrize("graph", ["cycle", "complete"])
def test_fused_local_dsgd_with_one_step_is_fused_dsgd_bitwise(graph):
    from test_gpu_mnist import _problem
    G = {"cycle": nx.cycle_graph(5), "complete": nx.complete_graph(5)}[graph]
    conf = dict(KG, local_steps=1, correction=False, alpha=0.02)
    dconf = {"alg_name": "dsgd", "alpha0": 0.02, "mu": 0.0, "outer_iterations": 7, "profile": False}
    a = _problem(5, 32, "fused", conf, graph=G, eval_every=3)
    b = _problem(5, 32, "fused", dconf, graph=G, eval_every=3)
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = KGT(a, DEV, copy.deepcopy(conf)), DSGD(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert oa._program.eng.sum_mode == (graph == "complete")
    assert torch.equal(a.arena.theta, b.arena.theta)
    assert a.forward_cnt == b.forward_cnt


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    """Host-fed and staged rounds (K = 3 staged batches per round) train exactly like the resident pipeline."""
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(KG, local_steps=3, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = KGT(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.c.clone(), opt.y.clone(), pr.forward_cnt, pr.calls.copy()))
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert torch.equal(x, y)
    assert outs[0][3] == outs[1][3] and (outs[0][4] == outs[1][4]).all()


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", KG, graph=nx.wheel_graph(5), eval_every=3)
        opt = KGT(pr, DEV, copy.deepcopy(KG))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.c.clone(), opt.y.clone()))
    for run in outs[1:]:
        for x, y in zip(run, outs[0]):
            assert torch.equal(x, y)


@CORR
@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model, correction):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(KG, correction=correction, local_steps=3, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = KGT(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = KGT(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = KGT(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    if correction:
        assert torch.equal(o2.c, of.c) and torch.equal(o2.y, of.y)
    assert second.forward_cnt == full.forward_cnt


@CORR
def test_sequence_check_passes_on_a_link_drop_run(correction):
    """Link drops every round (several topology tables, isolated nodes) with ``debug_sequence_check``: no stale row is
    read, and the result matches the PyTorch ops walking the same graph sequence."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(KG, correction=correction)
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 7}
        pr._init_faults()
        c = dict(copy.deepcopy(conf), debug_sequence_check=True,
                 consensus_backend="auto" if backend == "fused" else "torch")
        opt = KGT(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
