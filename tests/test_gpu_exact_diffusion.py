"""Exact Diffusion on the fused sm_90a kernels: ``ed_mix`` (``dsgd_mix_kernel`` with the weights of A = (I + W) / 2, or
``ed_sum_mix_kernel`` on the complete graph) and ``ed_step_kernel``, one launch at a time against a float64 oracle with
the bound of ``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err), then whole runs against the PyTorch path,
determinism, CUDA-graph replay and checkpoint/resume."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
from test_gpu_consensus_kernels import EXACT_GRAPHS, GRAPHS, S_LIST, VEC, KernelProblem, _snap
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import ExactDiffusion
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# every degree 0..9 appears: isolated (0..3), wheel5 (hub 4), star8 (hub 8), wheel10 (hub 9), random (5..7)
ED_GRAPHS = dict(GRAPHS, wheel5_ptr=[nx.wheel_graph(5)])
ROUNDS, CHECKED = 6, (0, 1, 5)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:10s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ oracle ----
def oracle_mix(st, *, k, nbrs, W, u, sum_mode, sums):
    """theta_i <- sum_j A_ij theta_j with A = (I + W) / 2 (own row live, neighbors published); complete graph:
    (theta_i + S / N) / 2 evaluated in float64 and rounded once."""
    N = st["theta"].shape[0]
    A = 0.5 * (np.eye(N) + W)
    out = dict(st, theta=st["theta"].copy())
    err = {"theta": np.zeros_like(st["theta"])}
    for i in range(N):
        if sum_mode:
            x = 0.5 * (st["theta"][i] + sums[0][0] / N)
            out["theta"][i] = x
            err["theta"][i] = u * np.abs(x) + co.U64 * 2.0 * (np.abs(st["theta"][i]) + np.abs(sums[0][0]) / N) + 0.5 * sums[1][0] / N
        else:
            out["theta"][i], err["theta"][i] = co._mix(i, st["theta"][i], st["pub"][k & 1, 0], nbrs, A, u)
    return out, err


def oracle_step(st, *, k, alpha, u):
    """psi' = theta - alpha g; theta <- psi' + (theta - psi) with psi = theta in round 0; psi <- psi'; theta published
    into the other parity."""
    par = k & 1
    g, e_g = co.sum_partials(st["grad_part"], u)
    th = st["theta"]
    ps = th if k == 0 else st["psi"]
    pn = th - alpha * g
    e_pn = alpha * e_g + u * (np.abs(th) + 2.0 * alpha * np.abs(g))
    dc = th - ps
    tn = pn + dc
    e_tn = e_pn + u * np.abs(dc) + u * np.abs(tn)
    pub, e_pub = st["pub"].copy(), np.zeros_like(st["pub"])
    pub[par ^ 1, 0], e_pub[par ^ 1, 0] = tn, e_tn
    return dict(st, theta=tn, psi=pn, pub=pub), {"theta": e_tn, "psi": e_pn, "pub": e_pub}


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, S, n, n_pad=None, seed=0, zero_cols=None, theta=None, mu=2.0):
    graphs = ED_GRAPHS[graph_key] if graph_key in ED_GRAPHS else EXACT_GRAPHS[graph_key]
    conf = {"alg_name": "exact_diffusion", "alpha0": 0.08, "mu": mu, "outer_iterations": ROUNDS, "profile": False}
    if graph_key.endswith("_ptr"):
        conf["complete_graph_mode"] = "pointer"
    pr = KernelProblem(graphs, n, dtype, S, seed=seed, n_pad=n_pad, zero_cols=zero_cols, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    th = torch.randn(pr.N, n, generator=g, dtype=torch.float64) if theta is None else theta
    pr.arena.theta[:, :n] = th.to(dtype).to(DEV)
    o = ExactDiffusion(pr, DEV, conf)
    # psi holds garbage before round 0: the kernel must take psi = theta there, not read the row
    o.psi[:, :n] = (1e3 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    return pr, o, conf


def _state(pr, o, eng):
    s = _snap(pr, o, eng)
    s["psi"] = o.psi.detach().double().cpu().numpy().copy()
    return s


class Harness:
    def __init__(self, pr, o, conf):
        self.pr, self.o = pr, o
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        want = co.dsgd_alpha_table(conf["alpha0"], conf["mu"], o.oits)
        self.alpha = self.eng.alpha.cpu().double().numpy()
        np.testing.assert_allclose(self.alpha, want, rtol=2 * self.u + 1e-14, atol=0)
        self.n = max(s.offset + s.numel for s in pr.layout.slots)

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        assert after["done_ctr"] == 0, name
        ends = name == "ed_step"
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if ends else 0)), name
        for key in ("theta", "pub", "psi"):
            assert not after[key][..., self.n:].any(), f"{name}: padding of {key} written"
        if ends:
            assert np.array_equal(after["pub"][(k & 1) ^ 1, 0], after["theta"]), f"{name}: pub[par^1] != theta"
        if not check:
            return
        tp = Topology(self.pr.plan_graphs(self.o.oits, 0, 1)[k])
        if name == "local_sum":
            s, e = co.local_sum(before["pub"], k & 1)
            want, err = dict(before, sum_local=before["sum_local"].copy()), {"sum_local": np.zeros_like(before["sum_local"])}
            want["sum_local"][k & 1], err["sum_local"][k & 1] = s, e
        elif name == "ed_mix":
            sums = None
            if self.eng.sum_mode:
                s = before["sum_local"][k & 1]
                sums = (s, co.U64 * np.abs(s))
            want, err = oracle_mix(before, k=k, nbrs=tp.neighbors_noself, W=tp.W, u=self.u,
                                   sum_mode=self.eng.sum_mode, sums=sums)
        else:
            want, err = oracle_step(before, k=k, alpha=self.alpha[k], u=self.u)
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name} round {k} {key}", got, want[key], err[key], C)
                WORST[(name, self.dt)] = max(WORST[(name, self.dt)], r)
            else:
                assert np.array_equal(got, before[key]), f"{name} wrote {key}"

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            if self.eng.sum_mode:
                self.launch("local_sum", op.local_sum, k, check=chk)
            self.launch("ed_mix", op.ed_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("ed_step", op.ed_step, k, check=chk)
        self.eng.check()


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(ED_GRAPHS))
def test_launches_match_oracle(graph_key, dtype):
    """Every graph (degrees 0-9, complete graph in sum and pointer mode, a graph that changes every round), rows of 13
    parameters (padding in the row), S rotating with the case; round 0 starts from a garbage psi row."""
    i = sorted(ED_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], n=13, seed=i)
    h = Harness(pr, o, conf)
    assert h.eng.sum_mode == graph_key.endswith("_sum")
    h.run()


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The 4-deep and 16-deep partial sums and the tail loop past 16 (degree-9 hub: both neighbor groups)."""
    pr, o, conf = _setup("wheel10", dtype, S, n=77, seed=S)
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    """A row of exactly one vector, and rows long enough that the grid is capped at the resident CTAs and every
    thread walks the row more than once (the pre-wait loads only on the first iteration)."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, conf = _setup("random5to7", dtype, 5, n=vec, n_pad=vec, seed=3)
        Harness(pr, o, conf).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, conf = _setup("random5to7", dtype, 17, n=140001, seed=4)
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("graph_key", ["complete8_ptr", "cubical"])
def test_consensus_is_a_fixed_point(graph_key, dtype):
    """All rows equal and a zero gradient on graphs whose weights of A are exact binary fractions (9/16 and 1/16,
    5/8 and 1/8): theta and psi stay on the row, bitwise."""
    N, n = EXACT_GRAPHS[graph_key][0].number_of_nodes(), 29
    row = torch.as_tensor(np.random.default_rng(1).integers(-512, 512, n) / 64.0)
    pr, o, conf = _setup(graph_key, dtype, 3, n=n, zero_cols=slice(None), theta=row.expand(N, n))
    h = Harness(pr, o, conf)
    assert not h.eng.sum_mode
    th0 = pr.arena.theta.clone()
    h.run(rounds=3, checked=(0, 1, 2))
    assert torch.equal(pr.arena.theta, th0)
    assert torch.equal(o.psi, th0)


@DTYPES
@pytest.mark.parametrize("graph_key", ["switch", "complete6_sum"])
def test_graph_replay_equals_eager_launches(graph_key, dtype):
    """A captured RoundProgram gives, round after round, bitwise the state of the eager launches."""
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup(graph_key, dtype, 5, n=300, seed=2)
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
ED = {"alg_name": "exact_diffusion", "alpha0": 0.05, "mu": 0.01, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def test_mnist_fp64_paper_shape_matches_torch_fp64():
    """The float64 conv-net kernel at the paper shape with the fp64 consensus kernels under CUDA graphs against autograd
    and the PyTorch ops in float64: within 1e-9 after one round and 1e-8 over the run."""
    from test_gpu_mnist import _generic_problem
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(ED))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(ED))
    b.arena.theta.copy_(a.arena.theta)
    oa = ExactDiffusion(a, DEV, copy.deepcopy(ED))
    ob = ExactDiffusion(b, DEV, dict(copy.deepcopy(ED), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.run_rounds(1)
    ob.run_rounds(1)
    torch.cuda.synchronize()
    assert _rel(a.arena.theta, b.arena.theta) < 1e-9
    oa.train()
    ob.train()
    assert _rel(a.arena.theta, b.arena.theta) < 1e-8
    assert _rel(oa.psi, ob.psi) < 1e-8
    assert a.forward_cnt == b.forward_cnt


@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete"])
def test_mnist_fp32_matches_torch_ops(graph):
    """fp32 tensor-core MNIST kernel, fused round programs against the PyTorch consensus ops driving the same fused
    forward/backward, with the tolerance of the other algorithms' fp32 comparison."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    N = 5
    G = {"cycle": nx.cycle_graph(N), "wheel": nx.wheel_graph(N), "complete": nx.complete_graph(N)}[graph]
    a = _problem(N, 32, "fused", ED, graph=G, eval_every=3)
    b = _problem(N, 32, "fused", ED, graph=G, eval_every=3)
    b.arena.theta.copy_(a.arena.theta)
    oa = ExactDiffusion(a, DEV, copy.deepcopy(ED))
    ob = ExactDiffusion(b, DEV, dict(copy.deepcopy(ED), consensus_backend="torch"))
    oa.train()
    ob.train()
    assert oa._program.eng.sum_mode == (graph == "complete")
    _assert_mostly_close(a.arena.theta, b.arena.theta)
    _assert_mostly_close(oa.psi, ob.psi)
    assert a.forward_cnt == b.forward_cnt
    assert len(a.metrics["validation_loss"]) == len(b.metrics["validation_loss"]) == 3


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    """Host-fed and staged rounds train exactly like the resident pipeline."""
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(ED, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = ExactDiffusion(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.psi.clone(), pr.forward_cnt, pr.calls.copy()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][2] == outs[1][2] and (outs[0][3] == outs[1][3]).all()


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(ED))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(ED))
    b.arena.theta.copy_(a.arena.theta)
    oa = ExactDiffusion(a, DEV, copy.deepcopy(ED))
    ob = ExactDiffusion(b, DEV, dict(copy.deepcopy(ED), consensus_backend="torch"))
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
    b.arena.theta.copy_(a.arena.theta)
    for pr in (a, b):
        pr.conf["optimizer_config"] = copy.deepcopy(ED)
    oa = ExactDiffusion(a, DEV, copy.deepcopy(ED))
    ob = ExactDiffusion(b, DEV, dict(copy.deepcopy(ED), consensus_backend="torch"))
    oa.train()
    ob.train()
    assert oa._use_engine() and not ob._use_engine()
    _assert_mostly_close(a.arena.theta, b.arena.theta)
    assert a.forward_cnt == b.forward_cnt


def test_online_density_fp64_dynamic_graph_matches_torch_fp64(tmp_path):
    """The online problem (graph planned from the robot poses, changing over the run) in float64."""
    from test_gpu_mlp_f64 import _online_problem
    oc = dict(ED, alpha0=0.002, outer_iterations=9)
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    ref.arena.theta.copy_(fused.arena.theta)
    of = ExactDiffusion(fused, DEV, copy.deepcopy(oc))
    ExactDiffusion(ref, DEV, dict(copy.deepcopy(oc), consensus_backend="torch")).train()
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
        pr = _problem(5, 32, "fused", ED, graph=nx.wheel_graph(5), eval_every=3)
        opt = ExactDiffusion(pr, DEV, copy.deepcopy(ED))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.psi.clone()))
    for th, ps in outs[1:]:
        assert torch.equal(th, outs[0][0]) and torch.equal(ps, outs[0][1])


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(ED, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = ExactDiffusion(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = ExactDiffusion(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = ExactDiffusion(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.psi, of.psi)
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_on_a_link_drop_run():
    """Link drops every round (several topology tables, isolated nodes) with ``debug_sequence_check``: no stale row is
    read, and the result matches the PyTorch ops walking the same graph sequence."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        pr = _problem(6, 32, "fused", ED, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 6}
        pr._init_faults()
        c = dict(copy.deepcopy(ED), debug_sequence_check=True,
                 consensus_backend="auto" if backend == "fused" else "torch")
        opt = ExactDiffusion(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
