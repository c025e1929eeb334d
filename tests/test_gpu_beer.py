"""BEER on the fused sm_90a kernels: ``beer_mix`` and ``beer_step`` one launch at a time against the float64 oracle of
``tests/beer_oracle.py`` (|kernel - oracle| <= 16 u err), both code channels byte for byte against
``consensus_ref.choco_encode`` of the kernel's own differences, then whole runs against the PyTorch path, DSGT,
determinism, CUDA-graph replay, the input pipelines, checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import beer_oracle as bo
import choco_oracle as cho
import consensus_oracle as co
from test_gpu_consensus_kernels import EXACT_GRAPHS, GRAPHS, S_LIST, KernelProblem
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import BEER, DSGT
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# every degree 0..9; the complete graphs run through the pointer table (BEER has no sum mode)
BEER_GRAPHS = {k: v for k, v in GRAPHS.items() if k != "switch"}
BEER_GRAPHS["wheel5"] = [nx.wheel_graph(5)]
COMPRESSORS = ["none", "int8", "sign"]
ROUNDS, CHECKED = 6, (0, 1, 5)
ROWS = ("theta", "h", "s_h", "v", "g", "s_g", "m_old")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel, compressor and dtype (c = %d):" % C)
    for (kern, comp, dt), r in sorted(WORST.items()):
        print(f"  {kern:9s} {comp:5s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, comp, S, n, n_pad=None, seed=0, holes=False, gamma=0.6):
    graphs = BEER_GRAPHS[graph_key] if graph_key in BEER_GRAPHS else EXACT_GRAPHS[graph_key]
    conf = {"alg_name": "beer", "alpha": 0.08, "gamma": gamma, "compressor": comp, "outer_iterations": ROUNDS,
            "profile": False}
    pr = KernelProblem(graphs, n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
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
    o = BEER(pr, DEV, conf)
    return pr, o, conf


def _state(pr, o, eng):
    L, t = pr.N, lambda x: x.detach().double().cpu().numpy().copy()
    st = {n: t(pr.arena.theta if n == "theta" else getattr(o, n)) for n in ROWS}
    st.update({n + "_t": (pr.arena.theta if n == "theta" else getattr(o, n)).detach().cpu().clone()
               for n in ("theta", "h", "v", "g")})
    st.update(pub=eng.pub[:, :, :L].contiguous().view(torch.uint8).cpu().numpy().copy(),
              calls=pr.fused.calls.cpu().numpy().copy(), round_ctr=int(eng.round_ctr.item()),
              done_ctr=int(eng.done_ctr.item()), grad_part=t(pr.fused.grad_part))
    return st


class Harness:
    def __init__(self, pr, o, conf):
        self.pr, self.o = pr, o
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        assert not self.eng.sum_mode and self.eng.C == 2
        self.dtype = pr.dtype
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.comp = conf["compressor"]
        self.gamma = float(NPDT[pr.dtype](conf["gamma"]))
        self.alpha = self.eng.alpha.cpu().double().numpy()
        self.live = ref.choco_live(pr.layout).numpy()
        self.live_t = ref.choco_live(pr.layout)
        self.n_pad = pr.layout.n_pad

    def _decode_all(self, rows):
        out, rel = [], 0.0
        for r in rows:
            d, rel = cho.decode(r, self.comp, self.n_pad, NPDT[self.dtype], self.live)
            out.append(d)
        return np.stack(out), rel

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        par = k & 1
        dead = ~self.live
        assert after["done_ctr"] == 0, name
        ends = name == "beer_step"
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if ends else 0)), name
        for key in ROWS:
            assert not after[key][:, dead].any(), f"{name}: padding or hole of {key} written"
        key = (name, self.comp, self.dt)
        if name == "beer_mix":
            assert np.array_equal(after["pub"], before["pub"]), "beer_mix wrote a published row"
            for n in ("h", "v", "g", "m_old"):
                assert np.array_equal(after[n], before[n]), f"beer_mix wrote {n}"
            if not check:
                return
            tp = Topology(self.pr.plan_graphs(self.o.oits, 0, 1)[k])
            dh, rel = self._decode_all(before["pub"][par, 0])
            dg, _ = self._decode_all(before["pub"][par, 1])
            th, sh, sg, e_th, e_sh, e_sg = bo.mix(before["theta"], before["h"], before["s_h"], before["v"], before["s_g"],
                                                  dh, dg, tp.neighbors_noself, tp.W, self.gamma, self.alpha[k], self.u,
                                                  rel)
            WORST[key] = max(WORST[key], co.check(f"{name} round {k} s_h", after["s_h"], sh, e_sh, C),
                             co.check(f"{name} round {k} s_g", after["s_g"], sg, e_sg, C),
                             co.check(f"{name} round {k} theta", after["theta"], th, e_th, C))
            return
        # beer_step
        for n in ("theta", "s_h", "s_g"):
            assert np.array_equal(after[n], before[n]), f"beer_step wrote {n}"
        assert np.array_equal(after["pub"][par], before["pub"][par]), "beer_step wrote the parity being read"
        # bytes of both channels: choco_encode of the kernel's own differences theta - h_in and v_out - g_in; the
        # estimates take the decoded codes with one rounding
        for ch, x, est in ((0, "theta_t", "h_t"), (1, "v_t", "g_t")):
            codes, dec = ref.choco_encode(after[x] - before[est], self.comp, self.live_t)
            got = after["pub"][par ^ 1, ch][:, :codes.shape[1]]
            bad = np.nonzero((got != codes.numpy()).any(1))[0]
            assert bad.size == 0, f"{name} round {k}: channel {ch} code rows of nodes {bad.tolist()} differ"
            assert torch.equal(after[est], before[est] + dec), f"{name} round {k}: channel {ch} estimate"
        if not check:
            return
        gr, e_gr = co.sum_partials(before["grad_part"], self.u)
        v, e_v = bo.step_tracker(before["v"], before["g"], before["s_g"], before["m_old"], gr, e_gr, self.gamma, self.u)
        WORST[key] = max(WORST[key], co.check(f"{name} round {k} v", after["v"], v, e_v, C),
                         co.check(f"{name} round {k} m_old", after["m_old"], gr, e_gr, C))

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            self.launch("beer_mix", op.beer_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("beer_step", op.beer_step, k, check=chk)
        self.eng.check()


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
COMPS = pytest.mark.parametrize("comp", COMPRESSORS)


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@COMPS
@pytest.mark.parametrize("graph_key", sorted(BEER_GRAPHS))
def test_launches_match_oracle(graph_key, comp, dtype):
    """Degrees 0-9 (isolated node included), complete graphs through the pointer table, rows of 77 parameters with an
    alignment hole (dead elements inside a block), S rotating with the case."""
    i = sorted(BEER_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, comp, S_LIST[i % len(S_LIST)], n=77, seed=i, holes=True)
    Harness(pr, o, conf).run()


@DTYPES
@COMPS
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, comp, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8 (degree-9 hub: both neighbor pairs and the odd one)."""
    pr, o, conf = _setup("wheel10", dtype, comp, S, n=100, seed=S)
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@DTYPES
@COMPS
@pytest.mark.parametrize("size", ["one_unit", "grid_stride"])
def test_row_sizes_match_oracle(size, comp, dtype):
    """A row of one 128-element alignment unit (fewer threads than a CTA), and rows long enough that the grid is capped
    at the resident CTAs and every warp walks the row more than once (the pre-wait loads only on the first pass)."""
    if size == "one_unit":
        pr, o, conf = _setup("random5to7", dtype, comp, 5, n=128, seed=3)
        Harness(pr, o, conf).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pr, o, conf = _setup("random5to7", dtype, comp, 17, n=140001, seed=4)
    vec = ref.CHOCO_VEC[dtype]
    assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@DTYPES
@COMPS
def test_all_zero_blocks_stay_zero(comp, dtype):
    """theta = 0 and a zero gradient: every code is zero (scale 0, no division), and every row stays 0."""
    pr, o, conf = _setup("cycle6", dtype, comp, 3, n=200)
    pr.arena.theta.zero_()
    pr.fused.base.zero_()
    pr.fused.slope.zero_()
    h = Harness(pr, o, conf)
    h.run(rounds=3, checked=(0, 1, 2))
    assert not pr.arena.theta.any() and not any(getattr(o, n).any() for n in ROWS[1:])
    if comp != "sign":          # a zero sign code still has its bits set (v >= 0); its scales are 0
        assert not h.eng.pub.view(torch.uint8).any()


def test_a_changing_graph_is_refused():
    pr, o, conf = _setup("cycle6", torch.float64, "int8", 3, n=40)
    pr.graphs = GRAPHS["switch"]
    with pytest.raises(ValueError, match="beer needs a fixed graph"):
        ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))


@DTYPES
def test_graph_replay_equals_eager_launches(dtype):
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup("wheel10", dtype, "sign", 5, n=300, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        states = []
        for _ in range(4):
            prog.run(1)
            o.k += 1
            torch.cuda.synchronize()
            s = _state(pr, o, prog.eng)
            states.append({k: v for k, v in s.items() if isinstance(v, np.ndarray)})
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            assert np.array_equal(x, b[key]), f"round {k}: {key}"


# ------------------------------------------------------------------------------------------ whole runs ----
BE = {"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _conf(comp, **kw):
    return dict(copy.deepcopy(BE), compressor=comp, **kw)


def _pair(make, conf):
    a, b = make(conf, "fused"), make(conf, "torch")
    b.arena.theta.copy_(a.arena.theta)
    oa = BEER(a, DEV, copy.deepcopy(conf))
    ob = BEER(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    return a, b, oa, ob


def _mnist64(conf, backend):
    from test_gpu_mnist import _generic_problem
    return _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))


def _density64(conf, backend):
    from test_gpu_mlp_f64 import _density
    return _density(4, 500, M=700, backend=backend, opt_conf=copy.deepcopy(conf))


def _state_tensors(pr, o):
    return [pr.arena.theta] + [getattr(o, n) for n in BEER.STATE]


@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("model", ["mnist_paper_fp64", "density_fp64"])
def test_fp64_runs_match_torch_path(model, comp):
    """Whole fp64 runs, fused against autograd and the PyTorch BEER ops, within the 1e-8 whole-run bound.  The quantized
    part of both pending codes (int8 codes, sign words) is equal; the scales follow the differences, within the bound."""
    make = _mnist64 if model == "mnist_paper_fp64" else _density64
    a, b, oa, ob = _pair(make, _conf(comp))
    oa.train()
    ob.train()
    for name in ROWS:
        x, y = (a.arena.theta, b.arena.theta) if name == "theta" else (getattr(oa, name), getattr(ob, name))
        r = _rel(x, y)
        print(f"{model} {comp} {name}: rel {r:.2e}")
        assert r < 1e-8, name
    n_pad = a.arena.n_pad
    q = {"none": 0, "int8": n_pad, "sign": n_pad // 8}[comp]
    for name in ("code_h", "code_g"):
        diff = (getattr(oa, name)[:, :q] != getattr(ob, name)[:, :q]).nonzero()
        assert diff.numel() == 0, f"{name} differ at (node, byte) {diff[:8].tolist()}"
        dec = [ref.choco_decode(getattr(o, name), comp, n_pad, torch.float64, o.live) for o in (oa, ob)]
        assert _rel(dec[0], dec[1]) < 1e-8, name
    assert a.forward_cnt == b.forward_cnt


def _assert_invariants(opt, tol):
    """s_h + W dec(qh pending) == W h and s_g + W dec(qg pending) == W g to round-off: every code applied once."""
    pr, a = opt.pr, opt.arena
    W = torch.as_tensor(pr.topology().W, dtype=torch.float64, device=DEV)
    worst = 0.0
    for s, est, code in ((opt.s_h, opt.h, opt.code_h), (opt.s_g, opt.g, opt.code_g)):
        dec = ref.choco_decode(code, opt.compressor, a.n_pad, a.dtype, opt.live).double()
        want = W @ est.double()
        got = s.double() + W @ dec
        r = ((got - want).norm() / want.norm().clamp_min(1e-300)).item()
        assert r < tol, r
        worst = max(worst, r)
    return worst


@pytest.mark.parametrize("comp", COMPRESSORS)
def test_mnist_fp32_matches_torch_ops(comp):
    """fp32 tensor-core MNIST kernel: ``none`` within the fp32 tolerance of the other algorithms' comparison; int8 and
    sign (where an fp32 rounding can flip a code) keep the sum invariants on the device state.  Final validation losses
    of both paths are printed."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    conf = _conf(comp, outer_iterations=40, alpha=0.01)
    a = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=13)
    b = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=13)
    b.arena.theta.copy_(a.arena.theta)
    oa = BEER(a, DEV, copy.deepcopy(conf))
    ob = BEER(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    oa.train()
    ob.train()
    oa._program.sync_back()
    print(f"fp32 {comp}: validation loss fused {a.metrics['validation_loss'][-1].mean().item():.4f} "
          f"torch {b.metrics['validation_loss'][-1].mean().item():.4f}")
    if comp == "none":
        _assert_mostly_close(a.arena.theta, b.arena.theta)
    for o in (oa, ob):
        print(f"  invariant rel {_assert_invariants(o, 1e-4):.2e}")
    assert a.forward_cnt == b.forward_cnt


def test_none_with_gamma_one_equals_fused_dsgt_own_tracker():
    """compressor none, gamma 1, from a common starting row: BEER's iterates are DSGT's with own_tracker_step and no
    initial gradient draw (fp64 density problem, fused both)."""
    conf = _conf("none", gamma=1.0, outer_iterations=9)
    a = _density64(conf, "fused")
    dconf = {"alg_name": "dsgt", "alpha": conf["alpha"], "init_grads": False, "own_tracker_step": True,
             "update_graph": False, "outer_iterations": 9, "profile": False}
    b = _density64(dconf, "fused")
    a.arena.theta[:] = a.arena.theta[0].clone()
    b.arena.theta.copy_(a.arena.theta)
    oa = BEER(a, DEV, copy.deepcopy(conf))
    ob = DSGT(b, DEV, copy.deepcopy(dconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    r = _rel(a.arena.theta, b.arena.theta)
    rv = _rel(oa.v, ob.y)
    print(f"beer none gamma=1 vs dsgt own tracker: theta rel {r:.2e}, tracker rel {rv:.2e}")
    assert r < 1e-8 and rv < 1e-8


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        conf = _conf("int8")
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = BEER(pr, DEV, copy.deepcopy(conf))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append([t.clone() for t in _state_tensors(pr, opt)])
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0]))


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = _conf("sign", outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = BEER(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        opt._program.sync_back()
        assert opt._program.pipeline == pl
        outs.append(([t.clone() for t in _state_tensors(pr, opt)], pr.forward_cnt))
    assert all(torch.equal(x, y) for x, y in zip(outs[0][0], outs[1][0]))
    assert outs[0][1] == outs[1][1]


@pytest.mark.parametrize("model", ["mnist_fp32_int8", "density_fp64_sign"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    if model == "mnist_fp32_int8":
        from test_gpu_mnist import _problem
        conf = _conf("int8", outer_iterations=6)

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density
        conf = _conf("sign", outer_iterations=6)

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = BEER(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = BEER(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3 and o1.code_h.any() and o1.code_g.any()
    second = make()
    o2 = BEER(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and torch.equal(o2.code_h, o1.code_h) and torch.equal(o2.code_g, o1.code_g)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for n in BEER.STATE:
        assert torch.equal(getattr(o2, n), getattr(of, n)), n
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_on_a_beer_run():
    """``debug_sequence_check``: every neighbor code row read is tagged with the current round."""
    from test_gpu_mnist import _problem
    conf = _conf("sign", debug_sequence_check=True, outer_iterations=10)
    pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
    opt = BEER(pr, DEV, conf)
    opt.train()
    assert opt._program.eng.seq_buf is not None
    opt._program.eng.check()
