"""DP-DSGD / DECOR on the fused sm_90a kernels: every ``dp_norm`` and ``dp_step`` launch against float64 oracles (degrees
0-9, S in {1, 3, 5, 17}, padded and grid-stride rows, a graph that changes every round), the kernel's noise against the
host twin of the stream, norms and rows independent of the one-wave grid and of the node order, fused DSGD bit for bit with a clip above every
norm and no noise, whole fp64 runs against the PyTorch path with the same ledger, and a link-drop run with the sequence
check.

Bounds.
* ``dp_norm``: the kernel's ``sum g^2`` (partials in chunk order) within a relative ``16 n_pad 2^-53`` of the exact sum
  of the squares of ``g`` (the partials summed in T in partial order, as the kernel sums them).
* ``dp_step`` given the kernel's norm: ``c = 16`` times ``u_T (|theta| + 2 alpha (|f g| + |v|)) + alpha e_v`` per
  element, where ``e_v`` bounds the difference between the kernel's and the twin's noise (next point).
* The noise.  Both sides evaluate the same Philox words and the same 53-bit uniforms exactly; they differ only in
  ``log``, ``sqrt`` and ``sincospi``, each within a few ulp on the device (CUDA Programming Guide, double-precision
  functions: log 1 ulp, sincospi 2 ulp) and in NumPy (the quadrant reduction of ops/consensus_ref.py keeps ``cos(pi y)``
  within about 1 ulp absolute).  A normal is at most ``r <= sqrt(2 ln 2^53) < 8.6`` in magnitude, so each normal
  differs by at most ``8 * 8.6 * 2^-53`` absolute (8 ulp of r, with margin); the fp64 sums and products of ``v`` add
  ``(deg + 2) 2^-53 |v|``, and the fp32 arm rounds ``v`` once more (``2^-24 |v|``).  ``e_v`` is that sum, scaled by
  ``C z_dp + deg C z_pair``."""
import collections
import copy
import math

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
from test_gpu_consensus_kernels import GRAPHS, VEC, KernelProblem
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.optimizers import DSGD, DPDSGD
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
DP_GRAPHS = {k: v for k, v in GRAPHS.items() if k != "complete6_sum"}     # the complete graph runs through the table
ROUNDS = 4
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
NORMAL_ERR = 8 * 8.6 * 2.0 ** -53


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / bound per launch and dtype:")
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:10s} {dt:5s} {r:.3f}")


def _conf(**kw):
    return dict({"alg_name": "dp_dsgd", "alpha0": 0.08, "mu": 2.0, "clip_norm": 1.5, "noise_multiplier": 0.3,
                 "pair_noise_multiplier": 0.6, "noise_seed": 21, "outer_iterations": ROUNDS, "profile": False}, **kw)


def _setup(graphs, dtype, S, n, n_pad=None, seed=0, zero_grads=False, **kw):
    conf = _conf(**kw)
    pr = KernelProblem(graphs, n, dtype, S, seed=seed, n_pad=n_pad, conf=conf,
                       zero_cols=list(range(n)) if zero_grads else None)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, DPDSGD(pr, DEV, conf)


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def _g_T(gpart, dtype):
    """The partials summed in T in partial order (sum_partials)."""
    t = NPDT[dtype]
    g = gpart[0].astype(t)
    for s in range(1, gpart.shape[0]):
        g = (g + gpart[s].astype(t)).astype(t)
    return g.astype(np.float64)


def run_checked(pr, o, rounds=ROUNDS):
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert eng.dp and not eng.sum_mode and eng.C == 1
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    u = co.unit_roundoff(NPDT[pr.dtype])
    n, N, n_pad = pr.n, pr.N, pr.arena.n_pad
    live = ref.choco_live(pr.arena.layout).numpy()
    topos = [Topology(g) for g in pr.plan_graphs(o.oits, 0, 1)]
    src, op = pr.fused, eng.op
    pstride = eng.norm_part.numel() // N
    for k in range(rounds):
        op.dsgd_mix()
        src.launch()
        torch.cuda.synchronize()
        th1, gpart = _t(pr.arena.theta), _t(src.grad_part)
        op.dp_norm()
        torch.cuda.synchronize()
        parts = _t(eng.norm_part).reshape(N, pstride)
        op.dp_step()
        torch.cuda.synchronize()
        th2, pub2 = _t(pr.arena.theta), _t(eng.pub)
        alpha = float(eng.alpha[k].item())
        nch = -(-n_pad // (256 * VEC[pr.dtype]))
        t = topos[k]
        for l in range(N):
            g = _g_T(gpart[l], pr.dtype)
            exact = math.fsum(g * g)
            ss = 0.0
            for ch in range(nch):
                ss += parts[l, ch]
            r = abs(ss - exact) / max(16 * n_pad * 2.0 ** -53 * exact, 1e-300)
            assert r <= 1.0, f"round {k} node {l}: norm^2 {ss!r} vs {exact!r}"
            WORST[("dp_norm", dt)] = max(WORST[("dp_norm", dt)], r)
            f = ref.dp_clip_factor(ss, o.clip)
            nb = t.neighbors_noself[l]
            v = ref.dp_noise(o.key, k, l, nb, n_pad, o.cz_dp, o.cz_pair, live)
            fT = float(NPDT[pr.dtype](f))
            want = th1[l] - alpha * (fT * g + v)
            scale = o.cz_dp + len(nb) * o.cz_pair
            ev = scale * (NORMAL_ERR + (len(nb) + 2) * 2.0 ** -53 * 8.6) + (u * np.abs(v) if dt == "fp32" else 0.0)
            err = u * (np.abs(th1[l]) + 2 * alpha * (np.abs(fT * g) + np.abs(v))) + alpha * ev
            WORST[("dp_step", dt)] = max(WORST[("dp_step", dt)], co.check(f"round {k} node {l} step", th2[l], want, err, C))
        assert not th2[:, n:].any(), "padding of theta"
        assert np.array_equal(pub2[(k & 1) ^ 1, 0, :N], th2)
        assert int(eng.round_ctr.item()) == k + 1 and int(eng.done_ctr.item()) == 0
    eng.check()
    return eng


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(DP_GRAPHS))
def test_launches_match_oracle(graph_key, dtype):
    """Degrees 0-9 and a graph that changes every round, rows of 13 parameters (padding in the row), S in {1, 3, 5,
    17}; a clip that binds for some nodes and rounds and not others."""
    i = sorted(DP_GRAPHS).index(graph_key)
    pr, o = _setup(DP_GRAPHS[graph_key], dtype, [1, 3, 5, 17][i % 4], 13, seed=i, clip_norm=3.0)
    run_checked(pr, o)


@DTYPES
@pytest.mark.parametrize("size", ["one_vector", "padded", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    vec = VEC[dtype]
    if size == "one_vector":
        pr, o = _setup(DP_GRAPHS["random5to7"], dtype, 5, vec, n_pad=vec, seed=3)
    elif size == "padded":
        pr, o = _setup(DP_GRAPHS["random5to7"], dtype, 3, 3 * vec + 1, seed=5)
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        pr, o = _setup(DP_GRAPHS["random5to7"], dtype, 17, 140001, seed=4, clip_norm=50.0)
        assert pr.N * -(-pr.arena.n_pad // (256 * vec)) > 8 * sms
    run_checked(pr, o, rounds=2)


@DTYPES
@pytest.mark.parametrize("zs", [(1.0, 0.0), (0.0, 1.0), (0.7, 1.3)], ids=["local", "pair", "both"])
def test_noise_matches_the_host_twin(zs, dtype):
    """theta = 0, g = 0, alpha = 1: the step leaves theta = -v; within the stated bound of the twin's v, and with
    z_dp = 0 the network sum of the rows is 0 to rounding."""
    n = 4099
    pr, o = _setup(DP_GRAPHS["switch"], dtype, 1, n, seed=7, zero_grads=True, alpha0=1.0, mu=0.0,
                   noise_multiplier=zs[0], pair_noise_multiplier=zs[1])
    pr.arena.theta.zero_()
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    dt = "fp32" if dtype == torch.float32 else "fp64"
    live = ref.choco_live(pr.arena.layout).numpy()
    topos = [Topology(g) for g in pr.plan_graphs(o.oits, 0, 1)]
    for k in range(3):
        pr.arena.theta.zero_()
        eng.pub.zero_()               # the mix pulls zero rows: theta is 0 when the step starts
        eng.op.dsgd_mix()
        pr.fused.launch()
        eng.op.dp_norm()
        eng.op.dp_step()
        torch.cuda.synchronize()
        got = -_t(pr.arena.theta)
        for l in range(pr.N):
            nb = topos[k].neighbors_noself[l]
            v = ref.dp_noise(o.key, k, l, nb, pr.arena.n_pad, o.cz_dp, o.cz_pair, live)
            scale = o.cz_dp + len(nb) * o.cz_pair
            ev = scale * (NORMAL_ERR + (len(nb) + 2) * 2.0 ** -53 * 8.6) + (2.0 ** -24 * np.abs(v) if dt == "fp32" else 0)
            r = float(np.max(np.abs(got[l] - v) / np.maximum(ev, 1e-300)))
            assert r <= 1.0, f"round {k} node {l}: noise ratio {r}"
            WORST[("noise", dt)] = max(WORST[("noise", dt)], r)
        if zs[0] == 0.0 and dt == "fp64":
            assert np.abs(got.sum(0)).max() <= 4 * 8 * np.abs(got).max() * 2.0 ** -52
    eng.check()


@DTYPES
def test_norms_and_rows_do_not_depend_on_the_grid(dtype):
    """Node 0 of an edgeless graph of 2 and of 60 nodes (60 local nodes shrink the one-wave grid of every launch) starts
    from the same row with the same round-0 gradient and draws the same stream: its norm partials and its row after
    the step are equal bit for bit."""
    n = 70001
    outs = []
    for N in (2, 60):
        pr, o = _setup([nx.empty_graph(N)], dtype, 3, n, seed=11, clip_norm=5.0, noise_multiplier=0.5)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        eng.op.dsgd_mix()
        pr.fused.launch()
        eng.op.dp_norm()
        eng.op.dp_step()
        torch.cuda.synchronize()
        outs.append((_t(eng.norm_part)[:eng.norm_part.numel() // N], _t(pr.arena.theta)[0]))
        eng.check()
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


@DTYPES
def test_norms_and_rows_do_not_depend_on_the_node_order(dtype):
    """The engine launches the nodes in the order ``node_order`` gives (on more than one rank: nodes with remote
    neighbors first).  Here the same op runs once in identity order and once with a reversed ``node_order`` set by hand:
    every norm partial and every row is equal bit for bit over rounds with pairwise noise on a changing graph, since a
    CTA row's node (and so its global id, ``node0 + l``) comes from the table, not from its launch position."""
    outs = []
    for order in (None, "reversed"):
        pr, o = _setup(DP_GRAPHS["switch"], dtype, 3, 1037, seed=13, clip_norm=2.0)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        op, keep = eng.op, None
        if order is not None:
            keep = torch.arange(pr.N - 1, -1, -1, dtype=torch.int32, device=DEV)
            op = type(eng.op)(dict(eng._keep, node_order=keep.data_ptr()))
        parts = []
        for k in range(ROUNDS):
            op.dsgd_mix()
            pr.fused.launch()
            op.dp_norm()
            op.dp_step()
            torch.cuda.synchronize()
            parts.append(_t(eng.norm_part))
        assert int(eng.round_ctr.item()) == ROUNDS
        eng.check()
        outs.append((np.stack(parts), _t(pr.arena.theta)))
        del keep
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


# ------------------------------------------------------------------------------------------ whole runs ----
PC = {"alg_name": "dp_dsgd", "alpha0": 0.01, "mu": 0.001, "clip_norm": 0.5, "noise_multiplier": 0.02,
      "pair_noise_multiplier": 0.05, "outer_iterations": 7, "profile": False}
DC = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 7, "profile": False}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _pair(a, b, conf):
    b.arena.theta.copy_(a.arena.theta)
    return DPDSGD(a, DEV, copy.deepcopy(conf)), DPDSGD(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))


@pytest.mark.parametrize("model", ["mnist_fp32", "mnist_fp64", "density_fp64"])
def test_clip_above_every_norm_and_no_noise_is_fused_dsgd_bit_for_bit(model):
    R = 12
    conf = dict(PC, clip_norm=1e30, noise_multiplier=0.0, pair_noise_multiplier=0.0, outer_iterations=R)
    dconf = dict(DC, outer_iterations=R)
    if model.startswith("mnist"):
        from test_gpu_mnist import _generic_problem
        dt = torch.float32 if model == "mnist_fp32" else torch.float64
        a = _generic_problem((3, 5, 64), dt, "fused", B=32, N=5, eval_every=1000, conf=copy.deepcopy(conf))
        b = _generic_problem((3, 5, 64), dt, "fused", B=32, N=5, eval_every=1000, conf=copy.deepcopy(dconf))
    else:
        from test_gpu_mlp_f64 import _density
        a, b = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf)), _density(4, 500, M=700, opt_conf=copy.deepcopy(dconf))
    b.arena.theta.copy_(a.arena.theta)
    oa, ob = DPDSGD(a, DEV, copy.deepcopy(conf)), DSGD(b, DEV, copy.deepcopy(dconf))
    assert oa._use_engine() and ob._use_engine()
    oa.train()
    ob.train()
    assert torch.equal(a.arena.theta, b.arena.theta)
    assert oa.alph == ob.alph


def test_mnist_fp64_matches_torch_fp64_and_the_ledgers_agree():
    from test_gpu_mnist import _generic_problem
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(PC))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(PC))
    oa, ob = _pair(a, b, PC)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\nMNIST fp64: rel {r:.2e}")
    assert r < 1e-10
    assert a.forward_cnt == b.forward_cnt and oa.alph == ob.alph
    assert np.array_equal(oa.rho_eav, ob.rho_eav) and np.array_equal(oa.rho_all, ob.rho_all)


def test_density_fp64_matches_torch_fp64():
    from test_gpu_mlp_f64 import _density
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(PC))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(PC))
    oa, ob = _pair(a, b, PC)
    assert oa._use_engine()
    oa.train()
    ob.train()
    r = _rel(a.arena.theta, b.arena.theta)
    print(f"\ndensity fp64: rel {r:.2e}")
    assert r < 1e-10
    assert np.array_equal(oa.rho_eav, ob.rho_eav)


def test_link_drop_run_with_the_sequence_check():
    """Links drop every round: the edge streams and the ledger follow each round's graph; every pull reads a row tagged
    with its round, and the fused fp64 run equals the PyTorch ops to round-off, ledger included."""
    from test_gpu_mnist import _generic_problem
    outs = []
    for backend in ("fused", "torch"):
        conf = dict(PC, outer_iterations=10, debug_sequence_check=True,
                    consensus_backend="auto" if backend == "fused" else "torch")
        pr = _generic_problem((3, 5, 64), torch.float64, "fused" if backend == "fused" else "torch", B=32, N=6,
                              eval_every=1000, conf=copy.deepcopy(conf))
        pr.graph = nx.cycle_graph(6)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.4, "seed": 3, "from_round": 0, "to_round": 10}
        pr._init_faults()
        assert len({tuple(sorted(g.edges())) for g in pr.plan_graphs(10, 0, 1)}) > 3
        if outs:
            pr.arena.theta.copy_(outs[0][0])
        opt = DPDSGD(pr, DEV, copy.deepcopy(conf))
        theta0 = pr.arena.theta.clone()
        opt.train()
        outs.append((theta0, pr.arena.theta.clone(), opt.rho_eav.copy()))
        if backend == "fused":
            eng = opt._program.eng
            assert eng.seq_buf is not None and len(eng.topos) > 3
            torch.cuda.synchronize()
            assert int(eng.err.item()) == 0
            eng.check()
    r = _rel(outs[0][1], outs[1][1])
    print(f"\nlink drops fp64: rel {r:.2e}")
    assert r < 1e-10
    assert np.array_equal(outs[0][2], outs[1][2])
