"""Moniqua on the fused sm_90a kernels: every ``mq_mix`` and ``mq_step`` launch against the float64 oracle
(tests/moniqua_oracle.py) at degrees 0-9 and 16, both dtypes, every bit width, both bases, one-vector, padded and
grid-stride rows and rounds 0 and later; code rows byte-equal to ``mq_encode`` of the kernel's own theta; margin counts
equal to the oracle's on rows built to leave the bound; codes and rows independent of the one-wave grid and of the node
order; graph replay equal to eager; whole fp64 runs against the PyTorch path; the input pipelines, resume at an odd
round and the sequence check with link drops.

Bounds.
* ``mq_mix``: the oracle's fp64 expression is the kernel's, operation for operation (the decode, ``w (xhat_j - xhat_i)``
  rounded on its own, the sums in neighbor order); the bound allows ``8 (deg + 2) 2^-53`` of the magnitudes plus half
  an ulp of the arena dtype for the final rounding.
* ``mq_step``: ``c = 16`` times the unit round-off of the arena dtype of ``|theta| + |alpha g| (+ |psi|)``."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
import moniqua_oracle as mo
from test_gpu_consensus_kernels import GRAPHS, KernelProblem
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.optimizers import Moniqua
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
MQ_GRAPHS = {k: v for k, v in GRAPHS.items() if k != "complete6_sum"}
MQ_GRAPHS["complete17"] = [nx.complete_graph(17)]                       # degree 16
ROUNDS = 3
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
BITS = pytest.mark.parametrize("bits", ref.MQ_BITS)
BASES = pytest.mark.parametrize("base", ref.MQ_BASES)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / bound per launch and dtype:")
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:8s} {dt:5s} {r:.3f}")


def _conf(**kw):
    return dict({"alg_name": "moniqua", "alpha0": 0.05, "mu": 1.0, "bits": 8, "theta_bound": 0.5, "rounding_seed": 17,
                 "outer_iterations": ROUNDS + 1, "profile": False}, **kw)


def _pad(n):
    return -(-n // 128) * 128


def _setup(graphs, dtype, S, n, n_pad=None, seed=0, spread=0.1, **kw):
    """Rows ``centre + U(-spread, spread)``: every edge within ``2 spread``."""
    conf = _conf(**kw)
    pr = KernelProblem(graphs, n, dtype, S, seed=seed, n_pad=n_pad or _pad(n), conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    centre = torch.randn(n, generator=g, dtype=torch.float64) * 3
    th = centre + (torch.rand(pr.N, n, generator=g, dtype=torch.float64) * 2 - 1) * spread
    pr.arena.theta[:, :n] = th.to(dtype).to(DEV)
    return pr, Moniqua(pr, DEV, conf)


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def _g_T(gpart, dtype):
    t = NPDT[dtype]
    g = gpart[0].astype(t)
    for s in range(1, gpart.shape[0]):
        g = (g + gpart[s].astype(t)).astype(t)
    return g.astype(np.float64)


def _codes(eng, par, N, bits):
    return ref.mq_unpack(eng.pub[par, 0, :N].contiguous().view(torch.uint8).cpu(), bits).numpy()


def run_checked(pr, o, rounds=ROUNDS):
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert eng.mq and not eng.sum_mode and eng.C == 1 and eng.row_bytes == o.code_bytes
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    u = co.unit_roundoff(NPDT[pr.dtype])
    eps = float(np.finfo(NPDT[pr.dtype]).eps)
    N, bits = pr.N, o.bits
    topos = [Topology(g) for g in pr.plan_graphs(o.oits, 0, 1)]
    src, op = pr.fused, eng.op
    live = o.live
    for k in range(rounds):
        codes = _codes(eng, k & 1, N, bits)
        th0, m0 = _t(pr.arena.theta), o.margin.cpu().numpy().copy()
        op.mq_mix()
        torch.cuda.synchronize()
        th1 = _t(pr.arena.theta)
        t = topos[k]
        W = ref.ed_weights(t.W) if o.base == "exact_diffusion" else t.W
        w_rows = W.astype(NPDT[pr.dtype]).astype(np.float64)
        nbrs = [t.neighbors_noself[l] for l in range(N)]
        want, bound, hits = mo.mix(th0, codes, w_rows, nbrs, 0, o.B, bits, eps)
        WORST[("mq_mix", dt)] = max(WORST[("mq_mix", dt)], co.check(f"round {k} mix", th1, want, bound, 1))
        assert np.array_equal(o.margin.cpu().numpy() - m0, hits), f"round {k}: margin hits"
        psi0 = _t(o.psi) if o.psi is not None else None
        src.launch()
        torch.cuda.synchronize()
        gpart = _t(src.grad_part)
        op.mq_step()
        torch.cuda.synchronize()
        th2 = _t(pr.arena.theta)
        alpha = float(eng.alpha[k].item())
        for l in range(N):
            g = _g_T(gpart[l], pr.dtype)
            new, pn, err = mo.step(th1[l], None if psi0 is None else psi0[l], g, alpha, k == 0, u)
            WORST[("mq_step", dt)] = max(WORST[("mq_step", dt)], co.check(f"round {k} node {l} step", th2[l], new, err, C))
            if pn is not None:
                co.check(f"round {k} node {l} psi", _t(o.psi)[l], pn, err, C)
        # the published code row is mq_encode of the kernel's own theta, byte for byte
        want_rows = ref.mq_encode(pr.arena.theta, o.B, bits, o.key, k + 1, range(N), live)
        got_rows = eng.pub[(k & 1) ^ 1, 0, :N].contiguous().view(torch.uint8)
        assert torch.equal(got_rows, want_rows), f"round {k}: code rows"
        assert not th2[:, pr.n:].any(), "padding of theta"
        assert int(eng.round_ctr.item()) == k + 1 and int(eng.done_ctr.item()) == 0
    eng.check()
    return eng


# ------------------------------------------------------------------------------------------ per launch ----
@BASES
@BITS
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(MQ_GRAPHS))
def test_launches_match_oracle(graph_key, dtype, bits, base):
    """Degrees 0-9 and 16 and a graph that changes every round, rows of 1000 parameters (padding in the row),
    S in {1, 3, 5, 17}, rounds 0 to 2."""
    i = sorted(MQ_GRAPHS).index(graph_key)
    pr, o = _setup(MQ_GRAPHS[graph_key], dtype, [1, 3, 5, 17][i % 4], 1000, seed=i, bits=bits, base=base)
    run_checked(pr, o)


@BASES
@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype, base):
    """The shortest row (128: one vector for a few threads of one warp), a row whose parameters end mid-vector, and a
    row long enough that every thread loops."""
    if size == "one_vector":
        pr, o = _setup(MQ_GRAPHS["random5to7"], dtype, 5, 3, seed=3, bits=2, base=base)
    elif size == "padded":
        pr, o = _setup(MQ_GRAPHS["random5to7"], dtype, 3, 4 * 128 + 37, seed=5, bits=4, base=base)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o = _setup(MQ_GRAPHS["random5to7"], dtype, 17, 140001, seed=4, bits=8, base=base)
        assert pr.N * -(-pr.arena.n_pad // 1024) > 8 * sms
    run_checked(pr, o, rounds=2)


@BITS
@DTYPES
def test_margin_counts_equal_the_oracle_on_rows_past_the_bound(dtype, bits):
    """Rows spread over 3 theta_bound: many elements decode near or past the wrap boundary; the kernel counts the hits
    the oracle counts, node by node (ordinary input, checked as every other launch)."""
    pr, o = _setup(MQ_GRAPHS["wheel10"], dtype, 1, 3000, seed=9, bits=bits, spread=0.75, theta_bound=0.5)
    run_checked(pr, o, rounds=2)
    assert int(o.margin.sum()) > 0


@BITS
@DTYPES
def test_codes_and_rows_do_not_depend_on_the_grid(dtype, bits):
    """Node 0 of an edgeless graph of 2 and of 60 nodes (60 local nodes shrink the one-wave grid) starts from the same
    row with the same gradient: its code row and its row after the step are equal bit for bit."""
    outs = []
    for N in (2, 60):
        pr, o = _setup([nx.empty_graph(N)], dtype, 3, 70001, seed=11, bits=bits)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        eng.op.mq_mix()
        pr.fused.launch()
        eng.op.mq_step()
        torch.cuda.synchronize()
        outs.append((_t(pr.arena.theta)[0], eng.pub[1, 0, 0].view(torch.uint8).cpu().clone()))
        eng.check()
    assert np.array_equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@BASES
@DTYPES
def test_codes_and_rows_do_not_depend_on_the_node_order(dtype, base):
    outs = []
    for order in (None, "reversed"):
        pr, o = _setup(MQ_GRAPHS["switch"], dtype, 3, 1037, seed=13, bits=4, base=base)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        op, keep = eng.op, None
        if order is not None:
            keep = torch.arange(pr.N - 1, -1, -1, dtype=torch.int32, device=DEV)
            op = type(eng.op)(dict(eng._keep, node_order=keep.data_ptr()))
        codes = []
        for k in range(ROUNDS):
            op.mq_mix()
            pr.fused.launch()
            op.mq_step()
            torch.cuda.synchronize()
            codes.append(eng.pub[(k & 1) ^ 1, 0, :pr.N].view(torch.uint8).cpu().clone())
        eng.check()
        outs.append((torch.stack(codes), _t(pr.arena.theta), o.margin.cpu().clone()))
        del keep
    assert torch.equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][2], outs[1][2])


# ------------------------------------------------------------------------------------------ whole runs ----
PC = {"alg_name": "moniqua", "alpha0": 0.01, "mu": 0.001, "bits": 8, "theta_bound": 0.2, "outer_iterations": 9,
      "profile": False}
FLIP_LIMIT = 4


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _mnist64(conf, backend, **kw):
    from test_gpu_mnist import _generic_problem
    return _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=5, eval_every=3, conf=copy.deepcopy(conf), **kw)


def _density64(conf, backend):
    from test_gpu_mlp_f64 import _density
    return _density(4, 500, M=700, backend=backend, opt_conf=copy.deepcopy(conf))


def _compare(oa, ob, a, b, what):
    """Fused against the PyTorch path: code elements whose rounding decision flipped (theta within a few ulp of a
    threshold) are counted and held to FLIP_LIMIT; without a flip the rows agree to 1e-10 relative."""
    ca, cb = ref.mq_unpack(oa.code.cpu(), oa.bits), ref.mq_unpack(ob.code.cpu(), ob.bits)
    flips = int((ca != cb).sum())
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\n{what}: rel {r:.2e}, code flips {flips}")
    assert flips <= FLIP_LIMIT
    assert r < (1e-10 if flips == 0 else 1e-3)
    assert torch.equal(oa.margin.cpu(), ob.margin.cpu())
    assert a.metrics["moniqua_edge_gap"] == pytest.approx(b.metrics["moniqua_edge_gap"], rel=1e-6)


@BASES
@pytest.mark.parametrize("model", ["mnist_fp64", "density_fp64"])
def test_fp64_runs_match_torch_path(model, base):
    make = _mnist64 if model == "mnist_fp64" else _density64
    conf = dict(PC, base=base)
    a, b = make(conf, "fused"), make(conf, "torch")
    b.arena.theta.copy_(a.arena.theta)
    oa = Moniqua(a, DEV, copy.deepcopy(conf))
    ob = Moniqua(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    _compare(oa, ob, a, b, f"{model} {base}")
    assert a.forward_cnt == b.forward_cnt and oa.alph == ob.alph


@pytest.mark.parametrize("no_graph", ["0", "1"])
def test_graph_replay_equals_eager_and_is_deterministic(monkeypatch, no_graph):
    outs = []
    for env in ("0", no_graph):
        monkeypatch.setenv("NNDT_NO_GRAPH", env)
        conf = dict(PC, base="exact_diffusion", bits=4)
        pr = _mnist64(conf, "fused")
        opt = Moniqua(pr, DEV, copy.deepcopy(conf))
        opt.train()
        assert opt._program.capturable == (env == "0")
        outs.append((pr.arena.theta.clone(), opt.code.clone(), opt.psi.clone(), opt.margin.clone()))
    assert all(torch.equal(x, y) for x, y in zip(*outs))


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(PC, theta_bound=0.5, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = Moniqua(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        opt._program.sync_back()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.code.clone(), opt.margin.clone(), pr.forward_cnt))
    assert all(torch.equal(x, y) for x, y in zip(outs[0][:3], outs[1][:3]))
    assert outs[0][3] == outs[1][3]


@BASES
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, base):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    from test_gpu_mnist import _problem
    conf = dict(PC, base=base, theta_bound=0.5, outer_iterations=6)

    def make():
        return _problem(4, 32, "fused", conf, M=100)
    full = make()
    of = Moniqua(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = Moniqua(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = Moniqua(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and torch.equal(o2.code, o1.code)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.code, of.code) and torch.equal(o2.margin, of.margin)
    if base == "exact_diffusion":
        assert torch.equal(o2.psi, of.psi)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt


def test_link_drop_run_with_the_sequence_check():
    """Links drop every round: every pull reads a code row tagged with its round, and the fused fp64 run equals the
    PyTorch ops (code flips counted as in the whole-run tests)."""
    from test_gpu_mnist import _generic_problem
    runs, theta0 = [], None
    for backend in ("fused", "torch"):
        conf = dict(PC, outer_iterations=10, debug_sequence_check=True,
                    consensus_backend="auto" if backend == "fused" else "torch")
        pr = _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=6, eval_every=1000, conf=copy.deepcopy(conf))
        pr.graph = nx.cycle_graph(6)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.4, "seed": 3, "from_round": 0, "to_round": 10}
        pr._init_faults()
        assert len({tuple(sorted(g.edges())) for g in pr.plan_graphs(10, 0, 1)}) > 3
        if theta0 is None:
            theta0 = pr.arena.theta.clone()
        pr.arena.theta.copy_(theta0)
        opt = Moniqua(pr, DEV, copy.deepcopy(conf))
        opt.train()
        runs.append((pr, opt))
        if backend == "fused":
            eng = opt._program.eng
            assert eng.seq_buf is not None and len(eng.topos) > 3
            torch.cuda.synchronize()
            assert int(eng.err.item()) == 0
            eng.check()
    (a, oa), (b, ob) = runs
    _compare(oa, ob, a, b, "link drops fp64")
