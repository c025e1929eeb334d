"""The consensus kernels (``ops/csrc/consensus.cu``) one launch at a time against the float64 oracle of
``tests/consensus_oracle.py``.

A real ``ConsensusEngine`` is built on a minimal problem whose gradient source fills the partial rows with seeded
values.  Every launch is issued eagerly; before and after it the whole device state is read back (theta, both
parities of the published rows, dual / delta / m / v, g_old, the complete-graph sums, the round and arrival
counters, the draw counters) and compared with the oracle applied to the state before: written arrays within
``C * err`` of the oracle coordinate by coordinate, everything else bitwise unchanged.  The worst error / bound ratio
per kernel and dtype is printed at the end of the module (``-s``)."""
import collections
import functools

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import DiNNO, DSGD, DSGT
from nn_distributed_training_b200.parallel.arena import FlatLayout, NodeArena, ParamSlot
from nn_distributed_training_b200.parallel.context import DistContext, Placement
from nn_distributed_training_b200.problems.base import ConsensusProblem
from nn_distributed_training_b200.utils.graph_generation import Topology, TopologyCache

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16                       # roundings on the longest path of one launch
VEC = {torch.float32: 4, torch.float64: 2}
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:14s} {dt:8s} {r:.3f}")


def _random_graph_5_to_7():
    for seed in range(10000):
        g = nx.gnp_random_graph(10, 0.6, seed=seed)
        d = [x for _, x in g.degree()]
        if min(d) == 5 and max(d) == 7:
            return g
    raise AssertionError("no seed gives degrees 5..7")


def _isolated():
    g = nx.Graph([(0, 1), (1, 2), (2, 3), (3, 0), (0, 2), (4, 5)])
    g.add_node(6)
    return nx.convert_node_labels_to_integers(g)


GRAPHS = {
    "path2_ptr": [nx.path_graph(2)],        # K2 is complete: degree 1 through the neighbor table
    "cycle6": [nx.cycle_graph(6)],
    "star8": [nx.star_graph(8)],
    "wheel10": [nx.wheel_graph(10)],
    "random5to7": [_random_graph_5_to_7()],
    "isolated": [_isolated()],
    "complete6_sum": [nx.complete_graph(6)],
    "complete6_ptr": [nx.complete_graph(6)],
    "switch": [nx.cycle_graph(6), nx.star_graph(5), nx.complete_graph(6), nx.path_graph(6), nx.empty_graph(6)],
}
# graphs whose Metropolis weights are powers of two (1/8, 1/4): mixing equal rows is exact
EXACT_GRAPHS = {"complete8_ptr": [nx.complete_graph(8)],
                "cubical": [nx.convert_node_labels_to_integers(nx.cubical_graph())]}
# (algorithm, optimizer, persistent moments, primal iterations) / DSGT: init_grads in the optimizer slot
ALGS = {
    "dinno-sgd": ("dinno", "sgd", False, 1), "dinno-adam": ("dinno", "adam", False, 3),
    "dinno-adamw": ("dinno", "adamw", False, 1), "dinno-adam-pers": ("dinno", "adam", True, 3),
    "dinno-adamw-pers": ("dinno", "adamw", True, 1), "dinno-sgd-3": ("dinno", "sgd", False, 3),
    "dsgd": ("dsgd", None, False, 1), "dsgt-init": ("dsgt", True, False, 1), "dsgt-noinit": ("dsgt", False, False, 1),
}
S_LIST = [1, 3, 4, 5, 16, 17, 40]
DECAYS = ["constant", "linear", "log"]
ROUNDS = 6                    # checked: 0, 1 and 5 (both parities, different table entries)
CHECKED = (0, 1, 5)


class GradSource:
    """Test-local stand-in for a fused forward/backward kernel: ``launch()`` writes ``base + calls * slope`` into the
    partial rows, seeded values that differ per node, per partial and per draw (the consensus kernels advance
    ``calls``), with zero padding.  All on the device, so it is capturable."""

    def __init__(self, L, S, n, n_pad, dtype, seed, zero_cols=None):
        g = torch.Generator().manual_seed(seed)
        sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
        # same sign across nodes and partials per coordinate, so |g| stays well above round-off
        base = sign * (0.5 + torch.rand(L, S, n, generator=g, dtype=torch.float64)) / S
        slope = sign * 0.1 * torch.rand(L, S, n, generator=g, dtype=torch.float64) / S
        if zero_cols is not None:
            base[..., zero_cols] = 0
            slope[..., zero_cols] = 0
        self.base = torch.zeros(L, S, n_pad, dtype=dtype, device=DEV)
        self.slope = torch.zeros(L, S, n_pad, dtype=dtype, device=DEV)
        self.base[..., :n] = base.to(dtype)
        self.slope[..., :n] = slope.to(dtype)
        self.grad_part = torch.zeros(L, S, n_pad, dtype=dtype, device=DEV)
        self.calls = torch.zeros(L, dtype=torch.int32, device=DEV)
        self.S = S
        self.dtype = dtype

    def launch(self):
        torch.addcmul(self.base, self.calls.view(-1, 1, 1).to(self.dtype), self.slope, out=self.grad_part)

    def sync_calls_from_host(self):
        self.calls.copy_(torch.as_tensor(self.pr_calls.astype(np.int32)))


class KernelProblem(ConsensusProblem):
    """Just what the engine and the round program read: placement, arena, topology and a gradient source."""

    def __init__(self, graphs, n, dtype, S, seed=0, n_pad=None, zero_cols=None, conf=None):
        self.device = torch.device(DEV)
        self.ctx = DistContext.single(self.device)
        self.graphs = graphs
        self.graph = graphs[0]
        self.N = self.graph.number_of_nodes()
        self.placement = Placement(self.N, 1, 0)
        self.dtype = dtype
        self.layout = FlatLayout([ParamSlot("w", (n,), 0, n)])
        if n_pad is not None:
            self.layout.n_pad = n_pad
        self.n = n
        self.arena = NodeArena(self.layout, self.N, self.device, dtype)
        self.conf = conf or {}
        self._topo_cache = TopologyCache()
        self._faults = None
        self.calls = np.zeros(self.N, dtype=np.int64)
        self.forward_cnt, self.train_batch_size = 0, 1
        self.fused = GradSource(self.N, S, n, self.layout.n_pad, dtype, seed, zero_cols)
        self.fused.pr_calls = self.calls

    def plan_graphs(self, oits, k0, draws_per_round, init_draws=0, refresh=True):
        return [self.graphs[k % len(self.graphs)] for k in range(oits)]


def _conf(alg, opt, persistent, pits, decay, graph_key):
    if alg == "dinno":
        c = {"alg_name": "dinno", "rho_init": 0.4, "rho_scaling": 1.3, "outer_iterations": ROUNDS,
             "primal_iterations": pits, "primal_optimizer": opt, "persistant_primal_opt": persistent,
             "primal_lr_start": 0.05, "primal_lr_finish": 0.004, "lr_decay_type": decay, "profile": False}
        if persistent and decay != "constant":
            c["persistent_follows_schedule"] = True
    elif alg == "dsgd":
        c = {"alg_name": "dsgd", "alpha0": 0.08, "mu": 2.0, "outer_iterations": ROUNDS, "profile": False}
    else:
        c = {"alg_name": "dsgt", "alpha": 0.03, "init_grads": opt, "outer_iterations": ROUNDS, "profile": False}
    if graph_key.endswith("_ptr"):
        c["complete_graph_mode"] = "pointer"      # complete graph through the neighbor table, not the network sum
    return c


def _setup(alg_key, graph_key, dtype, S, n, n_pad=None, decay="log", seed=0, zero_cols=None, theta=None):
    alg, opt, persistent, pits = ALGS[alg_key]
    conf = _conf(alg, opt, persistent, pits, decay, graph_key)
    graphs = GRAPHS[graph_key] if graph_key in GRAPHS else EXACT_GRAPHS[graph_key]
    pr = KernelProblem(graphs, n, dtype, S, seed=seed, n_pad=n_pad, zero_cols=zero_cols, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    th = torch.randn(pr.N, n, generator=g, dtype=torch.float64) if theta is None else theta
    pr.arena.theta[:, :n] = th.to(dtype).to(DEV)
    o = {"dinno": DiNNO, "dsgd": DSGD, "dsgt": DSGT}[alg](pr, DEV, conf)
    if alg == "dinno":
        o.duals[:, :n] = (0.1 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    return pr, o, conf


def _snap(pr, o, eng):
    L, t = pr.N, lambda x: x.detach().double().cpu().numpy().copy()
    s = dict(theta=t(pr.arena.theta), pub=t(eng.pub[:, :, :L]), grad_part=t(pr.fused.grad_part),
             calls=pr.fused.calls.cpu().numpy().copy(), round_ctr=int(eng.round_ctr.item()),
             done_ctr=int(eng.done_ctr.item()))
    if o.alg_name == "dinno":
        s.update(dual=t(o.duals), delta=t(o.delta), m=None if o.m is None else t(o.m), v=None if o.v is None else t(o.v))
    if o.alg_name == "dsgt":
        s["g_old"] = t(o.g)
    if eng.sum_mode:
        s["sum_local"] = t(eng.sum_buf.local)
    return s


class Harness:
    """Launch-by-launch driver: ``launch(name, fn, ...)`` snapshots, launches, snapshots and checks."""

    def __init__(self, pr, o, conf, eng=None):
        self.pr, self.o, self.conf = pr, o, conf
        self.eng = eng or ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        self.dtype = pr.dtype
        self.u = co.unit_roundoff(NPDT[pr.dtype])
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        # the device schedules against the equations (to the dtype's rounding); the per-launch oracle then takes the
        # values the kernel reads
        oits, tol = o.oits, 2 * self.u + 1e-14
        if o.alg_name == "dinno":
            tables = dict(rho=co.rho_table(conf, oits), lr=co.lr_table(conf, oits))
        elif o.alg_name == "dsgd":
            tables = dict(alpha=co.dsgd_alpha_table(conf["alpha0"], conf["mu"], oits))
        else:
            tables = dict(alpha=np.full(oits, float(conf["alpha"])))
        for name, want in tables.items():
            got = getattr(self.eng, name).cpu().double().numpy()
            np.testing.assert_allclose(got, want, rtol=tol, atol=0, err_msg=name)
            setattr(self, name, got)
        self.n = max(s.offset + s.numel for s in pr.layout.slots)     # end of the last parameter: padding after it
        self.worst = collections.defaultdict(float)

    def topo(self, k):
        return Topology(self.pr.plan_graphs(self.o.oits, 0, 1)[k])

    def _oracle(self, name, k, p, st):
        o, eng, u = self.o, self.eng, self.u
        tp = self.topo(k)
        sums = None
        if eng.sum_mode and name != "local_sum":
            s = st["sum_local"][k & 1]
            sums = (s, co.U64 * np.abs(s))
        kw = dict(k=k, nbrs=tp.neighbors_noself, u=u, sum_mode=eng.sum_mode, sums=sums)
        if name == "local_sum":
            s, e = co.local_sum(st["pub"], k & 1)
            want, err = st["sum_local"].copy(), np.zeros_like(st["sum_local"])
            want[k & 1], err[k & 1] = s, e
            return dict(st, sum_local=want), {"sum_local": err}
        if name == "dinno_update":
            return co.dinno_update(st, step=p, rho=self.rho[k], lr=self.lr[k], opt=o.opt_kind, pits=o.pits,
                                   persistent=o.persistent, dtype=NPDT[self.dtype], **kw)
        if name == "dsgd_mix":
            return co.dsgd_mix(st, W=tp.W, **kw)
        if name == "dsgd_step":
            return co.dsgd_step(st, k=k, alpha=self.alpha[k], u=u)
        if name == "dsgt_init":
            return co.dsgt_init(st, u=u)
        if name == "dsgt_mix":
            return co.dsgt_mix(st, W=tp.W, alpha=self.alpha[k], **kw)
        if name == "dsgt_track":
            return co.dsgt_track(st, W=tp.W, **kw)
        raise KeyError(name)

    def launch(self, name, fn, k, p=0, check=True):
        before = _snap(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _snap(self.pr, self.o, self.eng)
        if name == "grad":
            return after
        assert after["done_ctr"] == 0, name
        ends = name in ("dsgd_step", "dsgt_track") or (name == "dinno_update" and p == self.o.pits - 1)
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        consumes = name in ("dinno_update", "dsgd_step", "dsgt_init", "dsgt_track")
        assert np.array_equal(after["calls"], before["calls"] + (1 if consumes else 0)), name
        for key in ("theta", "pub", "dual", "delta", "m", "v", "g_old"):
            if after.get(key) is not None:
                assert not after[key][..., self.n:].any(), f"{name}: padding of {key} written"
        if name in ("dinno_update", "dsgd_step", "dsgt_track") and ends:
            par = k & 1
            assert np.array_equal(after["pub"][par ^ 1, 0], after["theta"]), f"{name}: pub[par^1] != theta"
        if not check:
            return after
        want, err = self._oracle(name, k, p, before)
        for key, got in after.items():
            if key in ("grad_part", "calls", "round_ctr", "done_ctr") or got is None:
                continue
            if key in err:
                r = co.check(f"{name} round {k} step {p} {key}", got, want[key], err[key], C)
                self.worst[name] = max(self.worst[name], r)
                WORST[(name, self.dt)] = max(WORST[(name, self.dt)], r)
            else:
                assert np.array_equal(got, before[key]), f"{name} wrote {key}"
        return after

    def round(self, k, check=True):
        o, op, src = self.o, self.eng.op, self.pr.fused
        if self.eng.sum_mode:
            self.launch("local_sum", op.local_sum, k, check=check)
        if o.alg_name == "dinno":
            for p in range(o.pits):
                self.launch("grad", src.launch, k)
                self.launch("dinno_update", functools.partial(op.dinno_update, p), k, p, check=check)
        elif o.alg_name == "dsgd":
            self.launch("dsgd_mix", op.dsgd_mix, k, check=check)
            self.launch("grad", src.launch, k)
            self.launch("dsgd_step", op.dsgd_step, k, check=check)
        else:
            self.launch("dsgt_mix", op.dsgt_mix, k, check=check)
            self.launch("grad", src.launch, k)
            self.launch("dsgt_track", op.dsgt_track, k, check=check)

    def run(self, rounds=ROUNDS, checked=CHECKED):
        if self.o.alg_name == "dsgt" and self.o.init_grads:
            self.launch("grad", self.pr.fused.launch, 0)
            self.launch("dsgt_init", self.eng.op.dsgt_init, 0)
        for k in range(rounds):
            self.round(k, check=k in checked)
        self.eng.check()


def _dtype_id(d):
    return "fp32" if d == torch.float32 else "fp64"


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=_dtype_id)


# ---------------------------------------------------------------------------------------------- tests ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(GRAPHS))
@pytest.mark.parametrize("alg_key", sorted(ALGS))
def test_launches_match_oracle(alg_key, graph_key, dtype):
    """Every algorithm on every graph: rows of 13 parameters (padding in the row), S and the lr decay rotating with
    the case so each value meets several algorithms."""
    i = sorted(ALGS).index(alg_key) + sorted(GRAPHS).index(graph_key)
    S, decay = S_LIST[i % len(S_LIST)], DECAYS[i % 3]
    pr, o, conf = _setup(alg_key, graph_key, dtype, S, n=13, decay=decay, seed=i)
    h = Harness(pr, o, conf)
    assert h.eng.sum_mode == graph_key.endswith("_sum")
    h.run()


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The 4-deep and 16-deep partial sums and the tail loop past 16, on the gradient-consuming kernel of each
    algorithm (degree-9 hub: both neighbor groups)."""
    for alg_key in ("dinno-adam", "dsgd", "dsgt-init"):
        pr, o, conf = _setup(alg_key, "wheel10", dtype, S, n=77, seed=S)
        Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("alg_key", ["dinno-adamw-pers", "dsgd", "dsgt-init"])
@pytest.mark.parametrize("size", ["one_vector", "grid_stride"])
def test_row_sizes_match_oracle(size, alg_key, dtype):
    """A row of exactly one vector, and rows long enough that the grid is capped at the resident CTAs and every
    thread walks the row more than once (the pre-wait prefetch only on the first iteration)."""
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o, conf = _setup(alg_key, "random5to7", dtype, 5, n=vec, n_pad=vec, seed=3)
        Harness(pr, o, conf).run()
        return
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 140001
    pr, o, conf = _setup(alg_key, "random5to7", dtype, 17, n=n, seed=4)
    L, n_pad = pr.N, pr.arena.n_pad
    assert L * -(-n_pad // (256 * vec)) > 8 * sms      # more CTAs than can ever be resident: >= 2 iterations
    Harness(pr, o, conf).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("alg_key", ["dinno-adam", "dinno-sgd", "dsgd", "dsgt-noinit"])
@pytest.mark.parametrize("graph_key", ["complete8_ptr", "cubical"])
def test_consensus_is_a_fixed_point(graph_key, alg_key, dtype):
    """All rows equal, zero duals, zero gradient, on graphs whose Metropolis weights are powers of two (1/8 and 1/4)
    so the mixed row is exact: DiNNO leaves theta unchanged with delta exactly 0, DSGD and DSGT reproduce the row,
    in both dtypes, bitwise."""
    N, n = EXACT_GRAPHS[graph_key][0].number_of_nodes(), 29
    row = torch.as_tensor(np.random.default_rng(1).integers(-512, 512, n) / 64.0)
    pr, o, conf = _setup(alg_key, graph_key, dtype, 3, n=n, zero_cols=slice(None), theta=row.expand(N, n))
    if o.alg_name == "dinno":
        o.duals.zero_()
    h = Harness(pr, o, conf)
    assert not h.eng.sum_mode
    th0 = pr.arena.theta.clone()
    h.run(rounds=3, checked=(0, 1, 2))
    assert torch.equal(pr.arena.theta, th0)
    if o.alg_name == "dinno":
        assert not o.delta.any()


@DTYPES
@pytest.mark.parametrize("alg_key", ["dinno-adam", "dinno-sgd"])
def test_zero_gradient_coordinates_take_no_step(alg_key, dtype):
    """Coordinates where every node agrees, the duals are 0 and the loss gradient is exactly 0 have g = 0 exactly:
    the first primal step must leave them bitwise unchanged (Adam: m = v = 0, the step is 0 / eps)."""
    n, zc = 40, slice(0, 40, 3)
    pr, o, conf = _setup(alg_key, "random5to7", dtype, 4, n=n, zero_cols=zc, seed=9)
    pr.arena.theta[:, zc] = pr.arena.theta[0, zc].clone()
    o.duals[:, zc] = 0
    h = Harness(pr, o, conf)
    th0 = pr.arena.theta[:, zc].clone()
    h.launch("grad", pr.fused.launch, 0)
    h.launch("dinno_update", functools.partial(h.eng.op.dinno_update, 0), 0, 0)
    assert torch.equal(pr.arena.theta[:, zc], th0)
    assert not o.delta[:, zc].any()


@DTYPES
@pytest.mark.parametrize("alg_key", ["dinno-adam-pers", "dsgd", "dsgt-init"])
@pytest.mark.parametrize("graph_key", ["switch", "complete6_sum"])
def test_graph_replay_equals_eager_launches(graph_key, alg_key, dtype):
    """A captured RoundProgram gives, round after round, bitwise the state of the eager launches."""
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup(alg_key, graph_key, dtype, 5, n=300, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
        if o.alg_name == "dsgt" and o.init_grads:
            prog.dsgt_init()
        o._initialised = True
        states = []
        for _ in range(4):
            prog.run(1)
            torch.cuda.synchronize()
            states.append(_snap(pr, o, prog.eng))
        assert bool(prog._graphs) == capture
        runs.append(states)
    for k, (a, b) in enumerate(zip(*runs)):
        for key, x in a.items():
            if isinstance(x, np.ndarray):
                assert np.array_equal(x, b[key]), f"round {k}: {key}"
            else:
                assert x == b[key], f"round {k}: {key}"


@DTYPES
def test_consensus_metric_matches_oracle(dtype):
    pr, o, conf = _setup("dsgd", "wheel10", dtype, 1, n=1000, seed=5)
    pr.arena.theta[3] = 2.5 * pr.arena.theta[2]
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    d_all, d_mean = eng.consensus_metric(0)
    (pair, e_pair), (mean, e_mean) = co.consensus_metric(pr.arena.theta.double().cpu().numpy())
    WORST[("metric", _dtype_id(dtype))] = max(co.check("pair", d_all.numpy(), pair, e_pair, C),
                                              co.check("mean", d_mean[:, 0].numpy(), mean, e_mean, C))


@pytest.mark.parametrize("perturb", ["affine", "square"])
def test_density_dinno_run_launches_match_oracle(perturb):
    """The float64 density DiNNO run of test_gpu_mlp_f64 (fused forward/backward, cycle of 4, Adam, 2 primal steps,
    7 rounds) launch by launch: every dinno_update within the per-launch bound, with the affine perturbation
    theta_l *= 1 + 0.03 l that once put the run at a round-off tie and with the quadratic one it uses now."""
    from test_gpu_mlp_f64 import DINNO, _density
    conf = dict(DINNO)
    pr = _density(4, 500, M=700, opt_conf=conf, perturb=False)
    for l in range(4):
        pr.arena.theta[l] *= 1.0 + 0.03 * (l if perturb == "affine" else l * l)
    o = DiNNO(pr, DEV, conf)
    h = Harness(pr, o, conf)
    h.run(rounds=conf["outer_iterations"], checked=range(conf["outer_iterations"]))
    print(f"\nRATIO density dinno {perturb}: {h.worst['dinno_update']:.3f}")
