"""DeTAG on the fused sm_90a kernels: ``ag_gossip_kernel`` at the first, a middle and the last sub-step (w = 1 and
w != 1) and ``detag_track_kernel`` at every partial depth, one launch at a time against the float64 oracle with the
bound of ``tests/consensus_oracle.py`` (|kernel - oracle| <= 16 u err), then whole runs against the PyTorch path and
against fused DSGT, the input pipelines, CUDA-graph replay across the 64-round capture boundary, determinism,
checkpoint/resume, the sequence check and the refusal of a changing graph."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import detag_oracle as do
from test_gpu_consensus_kernels import GRAPHS, S_LIST, VEC, KernelProblem, _snap
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import MAX_ROUNDS_PER_GRAPH, RoundProgram
from nn_distributed_training_b200.optimizers import DSGT, DeTAG
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# degrees 0..16 through the pointer table (DeTAG has no sum mode): isolated (0..3), path2 (1), random (5..7),
# complete6 (5), star8 (hub 8), wheel10 (hub 9), star16 (hub 16)
DT_GRAPHS = {k: v for k, v in GRAPHS.items() if k != "switch" and not k.endswith("_sum")}
DT_GRAPHS["star16"] = [nx.star_graph(16)]
ROUNDS, CHECKED = 4, (0, 1, 3)
ACC = pytest.mark.parametrize("accelerate", [True, False], ids=["chebyshev", "plain"])
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:22s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, S, n, K, accelerate, n_pad=None, seed=0):
    conf = {"alg_name": "detag", "alpha": 0.08, "gossip_steps": K, "accelerate": accelerate,
            "outer_iterations": ROUNDS, "profile": False}
    pr = KernelProblem(DT_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    rnd = lambda scale=1.0: (scale * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)  # noqa
    pr.arena.theta[:, :n] = rnd()
    o = DeTAG(pr, DEV, conf)
    # a nonzero start (as after a resume) exercises every term
    o.g_old[:, :n] = rnd()
    o.y[:, :n] = rnd()
    o.z[:, :n] = rnd()
    return pr, o, conf


def _state(pr, o, eng):
    s = _snap(pr, o, eng)
    t = lambda x: x.detach().double().cpu().numpy().copy()          # noqa: E731
    s["g_old"] = t(o.g_old)
    s["ymix"] = t(eng.ymix)
    return s


class Harness:
    def __init__(self, pr, o):
        self.pr, self.o = pr, o
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.K = o.gossip_steps
        self.omega = self.eng.omega.cpu().double().numpy()
        self.alpha = self.eng.alpha.cpu().double().numpy()
        assert len(self.alpha) == self.K * o.oits
        self.n = max(s.offset + s.numel for s in pr.layout.slots)
        # both parities hold rows: X_{s-1} of sub-step 1 is the other parity; ymix holds garbage until the last sub-step
        g = torch.Generator().manual_seed(7)
        N, n = pr.N, self.n
        par = 1
        self.eng.pub[par, :, :N, :n] = torch.randn(2, N, n, generator=g, dtype=torch.float64).to(pr.dtype).to(DEV)
        self.eng.ymix[:, :n] = (1e3 * torch.randn(N, n, generator=g, dtype=torch.float64)).to(pr.dtype).to(DEV)

    def launch(self, name, fn, k, s=0, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        p = self.K * k + s
        assert before["round_ctr"] == p, name
        assert after["done_ctr"] == 0, name
        ends = name == "detag_track" or s < self.K - 1
        assert after["round_ctr"] == p + (1 if ends else 0), name
        track = name == "detag_track"
        assert np.array_equal(after["calls"], before["calls"] + (1 if track else 0)), name
        for key in ("theta", "pub", "g_old", "ymix"):
            assert not after[key][..., self.n:].any(), f"{name}: padding of {key} written"
        if not check:
            return
        tp = Topology(self.pr.plan_graphs(self.o.oits, 0, 1)[k])
        if track:
            want, err = do.track(before, p=p, alpha=self.alpha[p], u=self.u)
            kern = "detag_track"
        else:
            want, err = do.gossip(before, p=p, s=s, K=self.K, omega=self.omega[s], nbrs=tp.neighbors_noself, W=tp.W,
                                  u=self.u)
            kern = f"ag_gossip {'last' if s == self.K - 1 else 'mid'} w{'=' if self.omega[s] == 1.0 else '!='}1"
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name}({s}) round {k} {key}", got, want[key], err[key], C)
                WORST[(kern, self.dt)] = max(WORST[(kern, self.dt)], r)
            else:
                assert np.array_equal(got, before[key]), f"{name}({s}) wrote {key}"

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            for s in range(self.K):
                self.launch("ag_gossip", lambda: op.ag_gossip(s), k, s=s, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("detag_track", op.detag_track, k, s=self.K - 1, check=chk)
        self.eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@ACC
@pytest.mark.parametrize("graph_key", sorted(DT_GRAPHS))
def test_launches_match_oracle(graph_key, accelerate, dtype):
    """Every graph (degrees 0-16), rows of 13 parameters (padding in the row), S and K rotating with the case: K = 3
    checks the first, a middle and the last sub-step, K = 2 a last one with w != 1 (accelerated), K = 1 DSGT's shape."""
    i = sorted(DT_GRAPHS).index(graph_key)
    K = (1, 2, 3)[i % 3]
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], 13, K, accelerate, seed=i)
    h = Harness(pr, o)
    assert h.eng.C == 2 and not h.eng.sum_mode
    if not accelerate:
        assert (h.omega == 1.0).all()
    h.run()


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The track kernel's 4-deep and 8-deep partial sums and the tail loop past 8 (degree-16 hub)."""
    pr, o, conf = _setup("star16", dtype, S, 77, 3, True, seed=S)
    Harness(pr, o).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    """A row of exactly one vector, and rows long enough that the grid is capped at the resident CTAs and every
    thread walks the row more than once."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, conf = _setup("random5to7", dtype, 5, vec, 3, True, n_pad=vec, seed=3)
        Harness(pr, o).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, conf = _setup("random5to7", dtype, 17, 140001, 3, True, seed=4)
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o).run(rounds=2, checked=(0, 1))


def test_a_changing_graph_is_refused():
    conf = {"alg_name": "detag", "alpha": 0.08, "gossip_steps": 2, "outer_iterations": 4, "profile": False}
    pr = KernelProblem(GRAPHS["switch"], 13, torch.float32, 1, conf=conf)
    o = DeTAG(pr, DEV, conf)
    with pytest.raises(ValueError, match="fixed graph"):
        ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    with pytest.raises(ValueError, match="fixed graph"):
        o.run_rounds(1)


# ------------------------------------------------------------------------------------------ whole runs ----
DT = {"alg_name": "detag", "alpha": 0.01, "gossip_steps": 3, "accelerate": True, "outer_iterations": 7,
      "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    oa = DeTAG(a, DEV, copy.deepcopy(conf))
    ob = DeTAG(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    return oa, ob


@ACC
def test_mnist_fp64_paper_shape_matches_torch_fp64(accelerate):
    """The float64 conv-net kernel at the paper shape with the fp64 consensus kernels under CUDA graphs against autograd
    and the PyTorch ops in float64, within the 1e-8 whole-run bound of the other algorithms."""
    from test_gpu_mnist import _generic_problem
    conf = dict(DT, accelerate=accelerate)
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64 accelerate={accelerate}: rel {r:.2e}")
    assert r < 1e-8
    assert _rel(oa.y, ob.y) < 1e-8 and _rel(oa.z, ob.z) < 1e-8
    assert a.forward_cnt == b.forward_cnt


@ACC
def test_density_fp64_matches_torch_fp64(accelerate):
    from test_gpu_mlp_f64 import _density
    conf = dict(DT, accelerate=accelerate)
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(conf))
    oa, ob = _pair(a, b, conf)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64 accelerate={accelerate}: rel {r:.2e}")
    assert r < 1e-8
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


def test_fused_one_gossip_step_is_fused_dsgt():
    """K = 1 on the fused kernels: theta and the tracker equal fused DSGT's (init_grads false) to rounding."""
    from test_gpu_mlp_f64 import _density
    conf = dict(DT, gossip_steps=1, outer_iterations=12)
    dconf = {"alg_name": "dsgt", "alpha": DT["alpha"], "init_grads": False, "outer_iterations": 12, "profile": False}
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, opt_conf=copy.deepcopy(dconf))
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = DeTAG(a, DEV, copy.deepcopy(conf)), DSGT(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    rx, ry = _rel(a.arena.theta, b.arena.theta), _rel(oa.y, ob.y)
    print(f"\nfused DeTAG K=1 vs fused DSGT: theta {rx:.2e}, trackers {ry:.2e}")
    assert rx < 1e-10 and ry < 1e-10


def test_graph_replay_across_the_capture_boundary_equals_eager_launches():
    """K = 3 over more rounds than one captured graph holds: the replayed graphs give bitwise the eager launches'
    state, and the device round counter ends at K times the gradient rounds."""
    from test_gpu_mnist import _problem
    R = MAX_ROUNDS_PER_GRAPH + 6
    outs = []
    for capture in (False, True):
        conf = dict(DT, outer_iterations=R)
        pr = _problem(5, 32, "fused", conf, graph=nx.cycle_graph(5), M=100, eval_every=1000)
        pr.conf["input_pipeline"] = "resident"
        opt = DeTAG(pr, DEV, copy.deepcopy(conf))
        prog = opt._program = RoundProgram(opt)
        prog.capturable = capture
        assert prog.launches_per_round() == 3 + 2
        opt.run_rounds(R)
        torch.cuda.synchronize()
        assert bool(prog._graphs) == capture
        assert int(prog.eng.round_ctr.item()) == 3 * R
        prog.eng.check()
        prog.sync_back()
        outs.append((pr.arena.theta.clone(), opt.y.clone(), opt.z.clone(), opt.g_old.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(DT, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = DeTAG(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.y.clone(), opt.z.clone(), pr.forward_cnt, pr.calls.copy()))
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert torch.equal(x, y)
    assert outs[0][3] == outs[1][3] and (outs[0][4] == outs[1][4]).all()


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic():
    from test_gpu_mnist import _problem
    outs = []
    for _ in range(2):
        pr = _problem(5, 32, "fused", DT, graph=nx.wheel_graph(5), eval_every=3)
        opt = DeTAG(pr, DEV, copy.deepcopy(DT))
        opt.train()
        outs.append((pr.arena.theta.clone(), opt.y.clone(), opt.z.clone(), opt.g_old.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(DT, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = DeTAG(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = DeTAG(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = DeTAG(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in ("y", "g_old", "z"):
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_with_three_gossip_steps():
    """``debug_sequence_check`` with K = 3: every sub-step reads rows tagged with its own protocol round, and the
    result matches the PyTorch ops."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(DT, debug_sequence_check=True, consensus_backend="auto" if backend == "fused" else "torch")
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        opt = DeTAG(pr, DEV, copy.deepcopy(conf))
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            eng = opt._program.eng
            assert eng.seq_buf is not None
            torch.cuda.synchronize()
            assert int(eng.err.item()) == 0
            eng.check()
    _assert_mostly_close(outs[0], outs[1])
