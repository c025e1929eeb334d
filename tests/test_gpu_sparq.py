"""SPARQ-SGD on the fused sm_90a kernels: ``sparq_mix``, ``sparq_step`` and ``sparq_publish`` one launch at a time
against the float64 oracle of ``tests/sparq_oracle.py`` (|kernel - oracle| <= 16 u err), code rows and tails byte for
byte against ``consensus_ref.choco_encode`` of the kernel's own v, a non-triggered neighbor's body never read (NaN
bodies change no bit), norm partials independent of the grid and the launch order, then graph replay, whole runs
against the PyTorch path, CHOCO-SGD at threshold 0 and local SGD above every error bit for bit, the input pipelines,
determinism, checkpoint/resume and the sequence check."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import choco_oracle as cho
import consensus_oracle as co
import sparq_oracle as so
from test_gpu_consensus_kernels import GRAPHS, KernelProblem
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import ChocoSGD, GossipPGA, SparqSGD

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
# degrees 0 .. 9 (an isolated node included) and a hub of 16
SPARQ_GRAPHS = {k: v for k, v in GRAPHS.items() if k not in ("switch", "complete6_sum")}
SPARQ_GRAPHS["wheel5"] = [nx.wheel_graph(5)]
SPARQ_GRAPHS["star16"] = [nx.star_graph(16)]
COMPRESSORS = ["none", "int8", "sign"]
S_LIST = [1, 3, 5, 17]
ROUNDS = 5


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel, compressor and dtype (c = %d):" % C)
    for (kern, comp, dt), r in sorted(WORST.items()):
        print(f"  {kern:14s} {comp:5s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, comp, S, n, H=1, seed=0, holes=False, threshold=0.0, n_pad=None):
    conf = {"alg_name": "sparq_sgd", "alpha0": 0.08, "mu": 2.0, "gamma": 0.6, "compressor": comp,
            "threshold": threshold, "local_steps": H, "outer_iterations": ROUNDS, "profile": False}
    pr = KernelProblem(SPARQ_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    if holes:
        from nn_distributed_training_b200.parallel.arena import FlatLayout, ParamSlot
        lay = FlatLayout([ParamSlot("a", (n // 2,), 0, n // 2), ParamSlot("b", (n - n // 2,), n // 2 + 3, n - n // 2)])
        pr.layout.slots, pr.layout.n = lay.slots, lay.n
    g = torch.Generator().manual_seed(seed + 1)
    live = ref.choco_live(pr.layout)
    th = torch.randn(pr.N, pr.layout.n_pad, generator=g, dtype=torch.float64) * live
    pr.arena.theta.copy_(th.to(dtype).to(DEV))
    pr.fused.base.mul_(live.to(DEV))
    pr.fused.slope.mul_(live.to(DEV))
    return pr, SparqSGD(pr, DEV, conf), conf


def _state(pr, o, eng):
    L, t = pr.N, lambda x: x.detach().double().cpu().numpy().copy()
    return dict(theta=t(pr.arena.theta), x_hat=t(o.x_hat), s=t(o.s),
                pub=eng.pub[:, 0, :L].contiguous().view(torch.uint8).cpu().numpy().copy(),
                calls=pr.fused.calls.cpu().numpy().copy(), round_ctr=int(eng.round_ctr.item()),
                done_ctr=int(eng.done_ctr.item()), grad_part=t(pr.fused.grad_part),
                norm=eng.norm_part.cpu().numpy().copy(), trig=o.triggers.cpu().numpy().copy(),
                theta_t=pr.arena.theta.detach().cpu().clone(), x_hat_t=o.x_hat.detach().cpu().clone())


class Harness:
    def __init__(self, pr, o, conf, mid=False):
        self.pr, self.o = pr, o
        self.eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, o.local_steps))
        self.dtype = pr.dtype
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.comp = conf["compressor"]
        self.gamma = float(NPDT[pr.dtype](conf["gamma"]))
        self.alpha = self.eng.alpha.cpu().double().numpy()
        self.live = ref.choco_live(pr.layout).numpy()
        self.live_t = ref.choco_live(pr.layout)
        self.n_pad = pr.layout.n_pad
        self.cb = o.code_bytes
        self.H = o.local_steps
        self.mid = mid            # set thr[k] between the two middle errors of the round: some trigger, some not
        self.nchunk = -(-self.n_pad // (256 * ref.CHOCO_VEC[pr.dtype]))
        self.pstride = self.eng.norm_part.numel() // pr.N
        self.decisions = []

    def _tails(self, rows):
        return np.array([so.tail(r, self.cb)[0] for r in rows], dtype=bool)

    def launch(self, name, fn, k, p=0, check=True):
        before = _state(self.pr, self.o, self.eng)
        if name == "sparq_publish" and self.mid:
            e = np.sort(before["norm"].reshape(self.pr.N, self.pstride)[:, :self.nchunk].sum(1))
            self.eng.sparq_thr[k] = float(0.5 * (e[len(e) // 2 - 1] + e[len(e) // 2])) if len(e) > 1 else 0.0
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        par = k & 1
        dead = ~self.live
        assert after["done_ctr"] == 0, name
        ends = name == "sparq_publish"
        draws = name == "sparq_publish" or (name == "sparq_step" and p < self.H - 1)
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if draws else 0)), name
        for key in ("theta", "x_hat", "s"):
            assert not after[key][:, dead].any(), f"{name}: padding or hole of {key} written"
        key = (name, self.comp, self.dt)
        if name == "sparq_mix":
            assert np.array_equal(after["pub"], before["pub"]) and np.array_equal(after["x_hat"], before["x_hat"])
            if not check:
                return
            tp = self.eng.topos[0]
            rows = before["pub"][par]
            trig = self._tails(rows)
            dec = np.stack([cho.decode(r, self.comp, self.n_pad, NPDT[self.dtype], self.live)[0] if t
                            else np.zeros(self.n_pad) for r, t in zip(rows, trig)])
            rel = 1.0 if self.comp == "int8" else 0.0
            th, sn, e_th, e_s = so.mix(before["theta"], before["x_hat"], before["s"], dec, trig, tp.neighbors_noself,
                                       tp.W, self.gamma, self.u, rel)
            WORST[key] = max(WORST[key], co.check(f"{name} round {k} s", after["s"], sn, e_s, C),
                             co.check(f"{name} round {k} theta", after["theta"], th, e_th, C))
            return
        if name == "sparq_step":
            assert np.array_equal(after["pub"], before["pub"]) and np.array_equal(after["x_hat"], before["x_hat"])
            assert np.array_equal(after["s"], before["s"])
            if not check:
                return
            g, e_g = co.sum_partials(before["grad_part"], self.u)
            th, e_th = so.step(before["theta"], g, e_g, self.alpha[k], self.u)
            r = co.check(f"{name}({p}) round {k} theta", after["theta"], th, e_th, C)
            if p == self.H - 1:       # the partials of (theta - x_hat)^2 summed in chunk order: the node's e
                got = after["norm"].reshape(self.pr.N, self.pstride)[:, :self.nchunk].sum(1)
                e, e_e = so.sqdist(after["theta"], after["x_hat"], self.u)
                r = max(r, co.check(f"{name} round {k} e", got, e, e_e, C))
            WORST[key] = max(WORST[key], r)
            return
        # sparq_publish
        assert np.array_equal(after["theta"], before["theta"]) and np.array_equal(after["s"], before["s"])
        assert np.array_equal(after["pub"][par], before["pub"][par]), "sparq_publish wrote the parity being read"
        thr = float(self.eng.sparq_thr[k].item())
        norm = before["norm"].reshape(self.pr.N, self.pstride)
        new = after["pub"][par ^ 1]
        v = after["theta_t"] - before["x_hat_t"]
        codes, dec = ref.choco_encode(v, self.comp, self.live_t)
        trig = np.zeros(self.pr.N, dtype=bool)
        for i in range(self.pr.N):
            e = 0.0
            for ch in range(self.nchunk):
                e += float(norm[i, ch])
            t, z, ei = so.tail(new[i], self.cb)
            assert z == 0 and ei == e, f"round {k} node {i}: tail e {ei} != the partials' sum {e}"
            assert bool(t) == (e > thr), f"round {k} node {i}"
            if thr > 0:
                assert abs(e - thr) > 1e-12 * thr, f"round {k} node {i}: a decision at the threshold"
            trig[i] = bool(t)
            if t:
                assert np.array_equal(new[i][:self.cb], codes[i].numpy()), f"round {k} node {i}: code != choco_encode"
                assert torch.equal(after["x_hat_t"][i], before["x_hat_t"][i] + dec[i])
            else:
                assert np.array_equal(new[i][:self.cb], before["pub"][par ^ 1][i][:self.cb]), "a body written"
                assert torch.equal(after["x_hat_t"][i], before["x_hat_t"][i])
        assert np.array_equal(after["trig"], before["trig"] + trig)
        self.decisions.append(trig)

    def run(self, rounds=ROUNDS, checked=(0, 1, ROUNDS - 1)):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            self.launch("sparq_mix", op.sparq_mix, k, check=chk)
            for p in range(self.H):
                self.launch("grad", src.launch, k)
                self.launch("sparq_step", lambda: op.sparq_step(p), k, p=p, check=chk)
            self.launch("sparq_publish", op.sparq_publish, k, check=chk)
        self.eng.check()
        return np.stack(self.decisions)


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
COMPS = pytest.mark.parametrize("comp", COMPRESSORS)


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@COMPS
@pytest.mark.parametrize("graph_key", sorted(SPARQ_GRAPHS))
def test_launches_match_oracle(graph_key, comp, dtype):
    """Degrees 0-9 and 16, rows of 77 parameters with an alignment hole, S and H rotating with the case, the threshold
    between the round's two middle errors (some nodes trigger and some do not)."""
    i = sorted(SPARQ_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, comp, S_LIST[i % len(S_LIST)], n=77, H=1 + i % 3, seed=i, holes=True)
    d = Harness(pr, o, conf, mid=True).run()
    if pr.N > 1:
        assert d.any() and not d.all()


@DTYPES
@COMPS
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_and_step_index_matches_oracle(S, comp, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8, three local steps (both step variants)."""
    pr, o, conf = _setup("wheel10", dtype, comp, S, n=100, H=3, seed=S)
    Harness(pr, o, conf, mid=True).run(rounds=2, checked=(0, 1))


@DTYPES
@COMPS
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, comp, dtype):
    """A row of one 128-element unit, a row padded past its parameters, and rows long enough that the grid is capped at
    the resident CTAs and every CTA walks several chunks."""
    if size == "one_vector":
        pr, o, conf = _setup("random5to7", dtype, comp, 5, n=128, H=2, seed=3)
    elif size == "padded":
        pr, o, conf = _setup("random5to7", dtype, comp, 3, n=130, H=1, seed=5, n_pad=512)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o, conf = _setup("random5to7", dtype, comp, 17, n=140001, H=2, seed=4)
        assert pr.N * -(-pr.arena.n_pad // (256 * ref.CHOCO_VEC[dtype])) > 8 * sms
    Harness(pr, o, conf, mid=True).run(rounds=2, checked=(0, 1))


@DTYPES
@COMPS
def test_a_non_triggered_neighbors_body_is_not_read(comp, dtype):
    """Before each mix, the code bodies of the rows whose tail says 0 are overwritten with 0xFF (NaN scales and values):
    the mix's s and theta are bit for bit those of the same mix on the intact bodies."""
    pr, o, conf = _setup("wheel10", dtype, comp, 3, n=300, H=1, seed=7)
    h = Harness(pr, o, conf, mid=True)
    op, src = h.eng.op, pr.fused
    seen = 0
    for k in range(4):
        par = k & 1
        theta0, s0 = pr.arena.theta.clone(), o.s.clone()
        op.sparq_mix()
        torch.cuda.synchronize()
        ref_out = (pr.arena.theta.clone(), o.s.clone())
        pr.arena.theta.copy_(theta0)
        o.s.copy_(s0)
        rows = h.eng.pub[par, 0, :pr.N].view(torch.uint8)
        trig, _ = ref.sparq_tail_read(rows.cpu(), h.cb)
        saved = rows.clone()
        rows[~trig.to(DEV), :h.cb] = 255
        seen += int((~trig).sum())
        op.sparq_mix()
        torch.cuda.synchronize()
        assert torch.equal(pr.arena.theta, ref_out[0]) and torch.equal(o.s, ref_out[1]), f"round {k}"
        rows.copy_(saved)
        src.launch()
        op.sparq_step(0)
        e = np.sort(h.eng.norm_part.view(pr.N, -1)[:, :h.nchunk].sum(1).cpu().numpy())
        h.eng.sparq_thr[k] = float(0.5 * (e[len(e) // 2 - 1] + e[len(e) // 2]))
        op.sparq_publish()
    torch.cuda.synchronize()
    assert seen > 0
    h.eng.check()


@DTYPES
def test_norm_partials_do_not_depend_on_the_grid_or_the_launch_order(dtype):
    """The same four node rows hosted among 4 and among 12 local nodes (different one-wave grids on a row long enough to
    cap them), and with the launch order reversed: the partials are equal bit for bit."""
    n = 140001
    conf = {"alg_name": "sparq_sgd", "alpha0": 0.08, "mu": 2.0, "gamma": 0.6, "compressor": "int8", "threshold": 0.0,
            "outer_iterations": ROUNDS, "profile": False}
    first = None
    out = []
    for N, reverse in ((4, False), (12, False), (12, True)):
        pr = KernelProblem([nx.cycle_graph(N)], n, dtype, 5, seed=9, conf=conf)
        if first is None:       # the rows of the first problem before its step
            g = torch.Generator().manual_seed(3)
            pr.arena.theta[:, :n] = torch.randn(N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
            first = [t[:4].clone() for t in (pr.arena.theta, pr.fused.base, pr.fused.slope)]
        else:
            for t, f in zip((pr.arena.theta, pr.fused.base, pr.fused.slope), first):
                t[:4].copy_(f)
        o = SparqSGD(pr, DEV, conf)
        o.x_hat[:, :n] = 0.25
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        order = None
        if reverse:
            order = torch.arange(N - 1, -1, -1, dtype=torch.int32, device=DEV)
            eng.op = type(eng.op)(dict(eng._keep, node_order=order.data_ptr()))
        pr.fused.launch()
        eng.op.sparq_step(0)
        torch.cuda.synchronize()
        out.append(eng.norm_part.view(N, -1)[:4].clone())
    assert torch.equal(out[0], out[1]) and torch.equal(out[0], out[2])


@DTYPES
def test_graph_replay_equals_eager_launches(dtype):
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup("wheel10", dtype, "sign", 5, n=300, H=2, seed=2, threshold=3.0)
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
        assert prog.launches_per_round() == 2 + 2 * 2
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            assert np.array_equal(x, b[key]), f"round {k}: {key}"


# ------------------------------------------------------------------------------------------ whole runs ----
SQ = {"alg_name": "sparq_sgd", "alpha0": 0.05, "mu": 0.01, "gamma": 0.5, "outer_iterations": 9, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _conf(comp, **kw):
    return dict(copy.deepcopy(SQ), compressor=comp, **kw)


def _mnist64(conf, backend):
    from test_gpu_mnist import _generic_problem
    return _generic_problem((3, 5, 64), torch.float64, backend, B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))


def _density64(conf, backend):
    from test_gpu_mlp_f64 import _density
    return _density(4, 500, M=700, backend=backend, opt_conf=copy.deepcopy(conf))


@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("model", ["mnist_paper_fp64", "density_fp64"])
def test_fp64_runs_match_torch_path(model, comp):
    """Whole fp64 runs with two local steps at a threshold where some node-rounds trigger: fused against autograd and
    the PyTorch ops within 1e-8, with equal trigger counts."""
    make = _mnist64 if model == "mnist_paper_fp64" else _density64
    conf = _conf(comp, threshold=2000.0, local_steps=2)
    a, b = make(conf, "fused"), make(conf, "torch")
    b.arena.theta.copy_(a.arena.theta)
    oa = SparqSGD(a, DEV, copy.deepcopy(conf))
    ob = SparqSGD(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    for name, x, y in (("theta", a.arena.theta, b.arena.theta), ("x_hat", oa.x_hat, ob.x_hat), ("s", oa.s, ob.s)):
        r = _rel(x, y)
        print(f"{model} {comp} {name}: rel {r:.2e}")
        assert r < 1e-8, name
    print(f"{model} {comp}: triggers {oa.triggers.tolist()} of {oa.k} rounds")
    assert torch.equal(oa.triggers, ob.triggers)
    assert a.forward_cnt == b.forward_cnt
    assert a.metrics["sparq_pulled_bytes"] == b.metrics["sparq_pulled_bytes"]


@DTYPES
@COMPS
def test_threshold_zero_is_fused_choco_bit_for_bit(comp, dtype):
    """Property 3 on the fused path: threshold 0 and one local step is fused CHOCO-SGD bit for bit."""
    from test_gpu_mnist import _generic_problem
    conf = _conf(comp, threshold=0.0, outer_iterations=12)
    cconf = {k: v for k, v in conf.items() if k != "threshold"} | {"alg_name": "choco_sgd"}
    a = _generic_problem((3, 5, 64), dtype, "fused", B=32, N=5, eval_every=5, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), dtype, "fused", B=32, N=5, eval_every=5, conf=copy.deepcopy(cconf))
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = SparqSGD(a, DEV, copy.deepcopy(conf)), ChocoSGD(b, DEV, copy.deepcopy(cconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    assert torch.equal(a.arena.theta, b.arena.theta) and torch.equal(oa.x_hat, ob.x_hat) and torch.equal(oa.s, ob.s)
    assert int(oa.triggers.sum()) == 12 * 5


@DTYPES
def test_a_threshold_above_every_error_is_fused_local_sgd(dtype):
    """Property 4 on the fused path: no trigger, so the run is Gossip-PGA's fused local SGD bit for bit (theta += 0
    would turn a -0 into +0: the zero parameters of the starting rows are set to 1e-3), and only tails are pulled."""
    from test_gpu_mnist import _generic_problem
    R = 10
    conf = _conf("int8", threshold=1e30, outer_iterations=R)
    lconf = {"alg_name": "gossip_pga", "alpha0": conf["alpha0"], "mu": conf["mu"], "period": R + 1, "gossip": False,
             "outer_iterations": R, "profile": False}
    a = _generic_problem((3, 5, 64), dtype, "fused", B=32, N=5, eval_every=4, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), dtype, "fused", B=32, N=5, eval_every=4, conf=copy.deepcopy(lconf))
    live = a.arena.theta[:, :a.layout.n]
    live[live == 0] = 1e-3           # no zero parameter (the biases start at 0)
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = SparqSGD(a, DEV, copy.deepcopy(conf)), GossipPGA(b, DEV, copy.deepcopy(lconf))
    oa.train()
    ob.train()
    assert oa._use_engine() and ob._use_engine()
    assert torch.equal(a.arena.theta, b.arena.theta)
    assert not oa.triggers.any() and oa.pulled_bytes() == 16 * R * int(a.topology().deg.sum())


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        conf = _conf("int8", threshold=2000.0, local_steps=2)
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = SparqSGD(pr, DEV, copy.deepcopy(conf))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.x_hat.clone(), opt.s.clone(), opt.code.clone(), opt.triggers.clone()))
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0]))


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = _conf("sign", threshold=2000.0, local_steps=2, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = SparqSGD(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        opt._program.sync_back()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.x_hat.clone(), opt.s.clone(), opt.code.clone(), opt.triggers.clone(),
                     pr.forward_cnt))
    assert all(torch.equal(x, y) for x, y in zip(outs[0][:5], outs[1][:5]))
    assert outs[0][5] == outs[1][5]


@pytest.mark.parametrize("model", ["mnist_fp32_int8", "density_fp64_sign"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    if model == "mnist_fp32_int8":
        from test_gpu_mnist import _problem
        conf = _conf("int8", threshold=2000.0, local_steps=2, outer_iterations=6)

        def make():
            return _problem(4, 32, "fused", conf, M=100)
    else:
        from test_gpu_mlp_f64 import _density
        conf = _conf("sign", threshold=2000.0, outer_iterations=6)

        def make():
            return _density(4, 300, M=500, opt_conf=conf)
    full = make()
    of = SparqSGD(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = SparqSGD(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = make()
    o2 = SparqSGD(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and torch.equal(o2.code, o1.code) and torch.equal(o2.triggers, o1.triggers)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for x, y in ((o2.x_hat, of.x_hat), (o2.s, of.s), (o2.triggers, of.triggers)):
        assert torch.equal(x, y)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_on_a_sparq_run():
    """``debug_sequence_check``: every neighbor row read (tail, and body when triggered) is tagged with the round."""
    from test_gpu_mnist import _problem
    conf = _conf("sign", threshold=2000.0, local_steps=2, debug_sequence_check=True, outer_iterations=10)
    pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
    opt = SparqSGD(pr, DEV, conf)
    opt.train()
    assert opt._program.eng.seq_buf is not None
    opt._program.eng.check()
