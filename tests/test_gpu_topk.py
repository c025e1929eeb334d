"""CHOCO-SGD and BEER with top-k codes on the fused sm_90a kernels: the sparse mix and the cluster step one launch at a
time against the float64 oracles (the harnesses of test_gpu_choco.py / test_gpu_beer.py, |kernel - oracle| <= 16 u
err), code rows byte for byte against ``consensus_ref.choco_encode`` of the kernel's own differences (ties, zero rows,
k = 1, k = n_live, last-ulp and signed-zero rows included), the capacity refusal, graph replay, whole runs against the
PyTorch path, ratio 1 against the compressor none, determinism, the input pipelines, checkpoint/resume and the sequence
check."""
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import topk_oracle as tko
import test_gpu_beer as gb
import test_gpu_choco as gc
from test_gpu_consensus_kernels import EXACT_GRAPHS, S_LIST, KernelProblem
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine, topk_max_row
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import BEER, ChocoSGD

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
GRAPHS = gc.CHOCO_GRAPHS
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
ALGS = pytest.mark.parametrize("alg", ["choco_sgd", "beer"])


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(alg, graph_key, dtype, S, n, ratio, seed=0, holes=False, gamma=0.6):
    graphs = GRAPHS[graph_key] if graph_key in GRAPHS else EXACT_GRAPHS[graph_key]
    if alg == "choco_sgd":
        conf = {"alg_name": "choco_sgd", "alpha0": 0.08, "mu": 2.0, "gamma": gamma}
    else:
        conf = {"alg_name": "beer", "alpha": 0.08, "gamma": gamma}
    conf.update(compressor="topk", topk_ratio=ratio, outer_iterations=gc.ROUNDS, profile=False)
    pr = KernelProblem(graphs, n, dtype, S, seed=seed, conf=conf)
    if holes:     # two parameter slots with an alignment hole between them: dead elements inside a block
        from nn_distributed_training_b200.parallel.arena import FlatLayout, ParamSlot
        lay = FlatLayout([ParamSlot("a", (n // 2,), 0, n // 2), ParamSlot("b", (n - n // 2,), n // 2 + 3, n - n // 2)])
        pr.layout.slots, pr.layout.n = lay.slots, lay.n
    g = torch.Generator().manual_seed(seed + 1)
    live = ref.choco_live(pr.layout)
    th = torch.randn(pr.N, pr.layout.n_pad, generator=g, dtype=torch.float64) * live
    pr.arena.theta.copy_(th.to(dtype).to(DEV))
    pr.fused.base.mul_(live.to(DEV))
    pr.fused.slope.mul_(live.to(DEV))
    o = (ChocoSGD if alg == "choco_sgd" else BEER)(pr, DEV, conf)
    return pr, o, conf


class _RefTopk:
    """consensus_ref with choco_encode bound to the optimizer's k: the harnesses encode the kernel's own differences
    with it and compare the code rows byte for byte."""

    def __init__(self, k):
        self.k = k

    def __getattr__(self, name):
        return getattr(ref, name)

    def choco_encode(self, v, compressor, live):
        return ref.choco_encode(v, compressor, live, self.k)


def _topk_harness(base):
    class H(base):
        def _decode_all(self, rows):
            return np.stack([tko.topk_decode(r, self.n_pad, NPDT[self.dtype], self.o.topk_k)[0] for r in rows]), 0.0
    return H


ChocoHarness, BeerHarness = _topk_harness(gc.Harness), _topk_harness(gb.Harness)


def _harness(alg, pr, o, conf, monkeypatch):
    mod = gc if alg == "choco_sgd" else gb
    monkeypatch.setattr(mod, "ref", _RefTopk(o.topk_k))
    return (ChocoHarness if alg == "choco_sgd" else BeerHarness)(pr, o, conf)


# ------------------------------------------------------------------------------------------ per launch ----
@ALGS
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(GRAPHS))
def test_launches_match_oracle(graph_key, dtype, alg, monkeypatch):
    """Degrees 0-9 (isolated node included), complete graphs through the pointer table, rows of 77 parameters with an
    alignment hole, S rotating with the case, k = 8 of 77."""
    i = sorted(GRAPHS).index(graph_key)
    pr, o, conf = _setup(alg, graph_key, dtype, S_LIST[i % len(S_LIST)], n=77, ratio=0.1, seed=i, holes=True)
    assert o.topk_k == 8
    _harness(alg, pr, o, conf, monkeypatch).run()


@ALGS
@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype, alg, monkeypatch):
    """The 4-deep and 8-deep partial sums (S <= 4 and > 4) on the degree-9 hub."""
    pr, o, conf = _setup(alg, "wheel10", dtype, S, n=300, ratio=0.05, seed=S)
    _harness(alg, pr, o, conf, monkeypatch).run(rounds=2, checked=(0, 1))


@ALGS
@DTYPES
@pytest.mark.parametrize("size", ["one_unit", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype, alg, monkeypatch):
    """A row of one 128-element unit (cluster CTAs without a slice), and rows long enough that the mix's grid is capped
    at the resident CTAs and loops over its chunks; the step's slices then hold thousands of keys per CTA."""
    if size == "one_unit":
        pr, o, conf = _setup(alg, "random5to7", dtype, 5, n=128, ratio=0.1, seed=3)
        _harness(alg, pr, o, conf, monkeypatch).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 100001 if dtype == torch.float64 else 140001
    pr, o, conf = _setup(alg, "random5to7", dtype, 17, n=n, ratio=0.01, seed=4)
    assert pr.N * -(-pr.arena.n_pad // (256 * ref.CHOCO_VEC[dtype])) > 8 * sms
    _harness(alg, pr, o, conf, monkeypatch).run(rounds=2, checked=(0, 1))


def _special_rows(N, n_pad, live, dtype):
    """Per node: heavy ties straddling the threshold, an all-zero row, values one ulp apart, -0 against +0 with a few
    nonzeros, random magnitudes; 0 on dead elements."""
    g = torch.Generator().manual_seed(9)
    idx = torch.arange(n_pad)
    one = torch.tensor(1.0, dtype=dtype)
    nxt = torch.nextafter(one, torch.tensor(2.0, dtype=dtype))
    rows = [torch.where(idx % 3 == 0, 2.0, -1.0).to(dtype),
            torch.zeros(n_pad, dtype=dtype),
            torch.where(idx % 2 == 1, nxt, one) * torch.where(idx % 5 == 2, -1.0, 1.0).to(dtype),
            torch.where(idx % 2 == 0, torch.tensor(-0.0, dtype=dtype), torch.tensor(0.0, dtype=dtype))]
    rows[3][[7, 100, 101]] = torch.tensor([3.0, -3.0, 1.0], dtype=dtype)
    while len(rows) < N:
        rows.append((torch.randn(n_pad, generator=g, dtype=torch.float64)
                     * torch.exp(4 * torch.randn(n_pad, generator=g, dtype=torch.float64))).to(dtype))
    return torch.stack(rows[:N]) * live.to(dtype)


@ALGS
@DTYPES
@pytest.mark.parametrize("ratio", ["k1", 0.3, 1.0])
def test_hard_rows_are_byte_equal_to_choco_encode(ratio, dtype, alg, monkeypatch):
    """A zero gradient and zero estimates make v the chosen rows: the code rows of the step are byte-equal to
    choco_encode (the harness's check), for k = 1, k = 30 % (inside the tie groups) and k = n_live."""
    r = 1e-9 if ratio == "k1" else ratio
    pr, o, conf = _setup(alg, "wheel5", dtype, 3, n=300, ratio=r, seed=1, holes=True)
    live = ref.choco_live(pr.layout)
    pr.arena.theta.copy_(_special_rows(pr.N, pr.layout.n_pad, live, dtype).to(DEV))
    pr.fused.base.zero_()
    pr.fused.slope.zero_()
    n_live = int(live.sum())
    assert o.topk_k == {"k1": 1, 0.3: 90, 1.0: n_live}[ratio]
    h = _harness(alg, pr, o, conf, monkeypatch)
    h.run(rounds=2, checked=(0, 1))


@ALGS
def test_a_row_beyond_the_cluster_shared_memory_is_refused(alg):
    limit = topk_max_row(8, 2 if alg == "beer" else 1)
    pr, o, conf = _setup(alg, "cycle6", torch.float64, 3, n=limit + 1000, ratio=0.01)
    with pytest.raises(ValueError, match=f"shared memory .*at most {limit} elements"):
        ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))


@ALGS
@DTYPES
def test_graph_replay_equals_eager_launches(dtype, alg):
    runs = []
    state = gc._state if alg == "choco_sgd" else gb._state
    for capture in (False, True):
        pr, o, conf = _setup(alg, "wheel10", dtype, 5, n=3000, ratio=0.02, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            s = state(pr, o, prog.eng)
            states.append({k: v for k, v in s.items() if isinstance(v, np.ndarray)})
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            assert np.array_equal(x, b[key]), f"round {k}: {key}"


# ------------------------------------------------------------------------------------------ whole runs ----
def _cls(alg):
    return ChocoSGD if alg == "choco_sgd" else BEER


def _conf(alg, **kw):
    base = gc.CH if alg == "choco_sgd" else gb.BE
    return dict(copy.deepcopy(base), **dict({"compressor": "topk", "topk_ratio": 0.01}, **kw))


def _rows_of(pr, o):
    return {"theta": pr.arena.theta, **{n: getattr(o, n) for n in o.STATE}}


@ALGS
@pytest.mark.parametrize("model", ["mnist_paper_fp64", "density_fp64"])
def test_fp64_runs_match_torch_path(model, alg):
    """Whole fp64 runs, fused against autograd and the PyTorch ops, within the 1e-8 whole-run bound.  Which entries a
    code row keeps depends on v to the last bit, so the rows are compared through what they decode to."""
    make = gc._mnist64 if model == "mnist_paper_fp64" else gc._density64
    conf = _conf(alg)
    a, b = make(conf, "fused"), make(conf, "torch")
    b.arena.theta.copy_(a.arena.theta)
    oa = _cls(alg)(a, DEV, copy.deepcopy(conf))
    ob = _cls(alg)(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    ra, rb = _rows_of(a, oa), _rows_of(b, ob)
    for name in ra:
        x, y = ra[name], rb[name]
        if name.startswith("code"):
            x, y = (ref.choco_decode(t, "topk", a.arena.n_pad, torch.float64, oa.live, oa.topk_k) for t in (x, y))
        r = gc._rel(x, y)
        print(f"{model} {alg} topk {name}: rel {r:.2e}")
        assert r < 1e-8, name
    assert a.forward_cnt == b.forward_cnt


@ALGS
def test_mnist_fp32_matches_torch_ops(alg):
    """fp32 tensor-core MNIST kernel: the sum invariants hold on the device state and on the PyTorch path's (an fp32
    rounding can change which entries a row keeps, so the runs are not compared element by element)."""
    from test_gpu_mnist import _problem
    conf = _conf(alg, outer_iterations=40)
    if alg == "beer":
        conf["alpha"] = 0.01
    a = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=13)
    b = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=13)
    b.arena.theta.copy_(a.arena.theta)
    oa = _cls(alg)(a, DEV, copy.deepcopy(conf))
    ob = _cls(alg)(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    oa.train()
    ob.train()
    oa._program.sync_back()
    print(f"fp32 {alg} topk: validation loss fused {a.metrics['validation_loss'][-1].mean().item():.4f} "
          f"torch {b.metrics['validation_loss'][-1].mean().item():.4f}")
    for o in (oa, ob):
        W = torch.as_tensor(o.pr.topology().W, dtype=torch.float64, device=DEV)
        pairs = [(o.s, o.x_hat, o.code)] if alg == "choco_sgd" else [(o.s_h, o.h, o.code_h), (o.s_g, o.g, o.code_g)]
        for s, est, code in pairs:
            dec = ref.choco_decode(code, "topk", o.arena.n_pad, o.arena.dtype, o.live, o.topk_k).double()
            want = W @ est.double()
            r = ((s.double() + W @ dec - want).norm() / want.norm().clamp_min(1e-300)).item()
            print(f"  invariant rel {r:.2e}")
            assert r < 1e-4
    assert a.forward_cnt == b.forward_cnt


@ALGS
@pytest.mark.parametrize("model", ["mnist_paper_fp64", "density_fp64"])
def test_ratio_one_is_bitwise_fused_none(model, alg):
    """topk_ratio 1 selects every live element with its exact value, and the sparse mix runs the dense mix's
    arithmetic: every row of the fused run is bitwise that of the fused compressor none."""
    make = gc._mnist64 if model == "mnist_paper_fp64" else gc._density64
    outs = []
    for comp in ("topk", "none"):
        conf = _conf(alg, topk_ratio=1.0) if comp == "topk" else dict(copy.deepcopy(gc.CH if alg == "choco_sgd" else gb.BE),
                                                                     compressor="none")
        pr = make(conf, "fused")
        if outs:
            pr.arena.theta.copy_(outs[0][0])
        o = _cls(alg)(pr, DEV, copy.deepcopy(conf))
        th0 = pr.arena.theta.clone()
        o.train()
        assert o._use_engine()
        outs.append([th0, pr.arena.theta.clone()] + [getattr(o, n).clone() for n in o.STATE if not n.startswith("code")])
    for x, y in zip(*outs):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------- determinism and resume ----
@ALGS
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(alg, monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        conf = _conf(alg)
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = _cls(alg)(pr, DEV, copy.deepcopy(conf))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append([t.clone() for t in _rows_of(pr, opt).values()])
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0]))


@ALGS
@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline, alg):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = _conf(alg, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = _cls(alg)(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        opt._program.sync_back()
        assert opt._program.pipeline == pl
        outs.append(([t.clone() for t in _rows_of(pr, opt).values()], pr.forward_cnt))
    assert all(torch.equal(x, y) for x, y in zip(outs[0][0], outs[1][0]))
    assert outs[0][1] == outs[1][1]


@ALGS
@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model, alg):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alg, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    cls = _cls(alg)
    full = make()
    of = cls(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = cls(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = cls(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and all(torch.equal(getattr(o2, n), getattr(o1, n)) for n in cls.STATE)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for n in cls.STATE:
        assert torch.equal(getattr(o2, n), getattr(of, n)), n
    assert second.forward_cnt == full.forward_cnt


@ALGS
def test_sequence_check_passes_on_a_topk_run(alg):
    """``debug_sequence_check``: every neighbor code row read is tagged with the current round."""
    from test_gpu_mnist import _problem
    conf = _conf(alg, debug_sequence_check=True, outer_iterations=10)
    pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
    opt = _cls(alg)(pr, DEV, conf)
    opt.train()
    assert opt._program.eng.seq_buf is not None
    opt._program.eng.check()
