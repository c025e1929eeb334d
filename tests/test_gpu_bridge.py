"""BRIDGE on the fused sm_90a kernels: ``bridge_mix_kernel`` and ``cg_step_kernel`` one launch at a time against the
float64 rules of ``tests/bridge_oracle.py`` (fp32 and fp64, degrees 0 to 9, the complete graph through the pointer
table, a graph that changes every round, padded and grid-stride rows, both screens, b from 0 to 3, every attack), the
screening guarantee on the kernel's output, independence of the neighbor table order, of the node order and of the
slot count, then whole runs: fp64 MNIST under each screen and attack against the PyTorch path, determinism, graph
replay, the input pipelines, resume and the sequence check with an ALIE attacker."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import bridge_oracle as bo
import consensus_oracle as co
from test_gpu_consensus_kernels import GRAPHS, KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.optimizers import Bridge
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16                      # bound multiplier, as tests/consensus_oracle.py
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
WORST = collections.defaultdict(float)
ROUNDS = 4
# Byzantine nodes per graph: adjacent attackers, an honest node whose only neighbor attacks (isolated: 4-5), an
# isolated attacker (6), the hub of the star and the wheel
BYZ = {"path2_ptr": [1], "cycle6": [0, 1], "star8": [0], "wheel10": [0, 5], "random5to7": [2],
       "isolated": [4, 6], "complete6_sum": [0, 1], "complete6_ptr": [0, 1], "switch": [1]}
U64 = 2.0 ** -53


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / bound per launch and dtype:")
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:22s} {dt:5s} {r:.3f}")


def _ratio(name, dt, got, want, err):
    r = float(np.max(np.abs(got - want) / err)) if got.size else 0.0
    WORST[(name, dt)] = max(WORST[(name, dt)], r)
    assert r <= 1.0, f"{name}: worst ratio {r:.3f}"


def _bconf(screen, b, **kw):
    c = {"alg_name": "bridge", "alpha0": 0.08, "mu": 0.5, "screen": screen, "outer_iterations": ROUNDS,
         "profile": False}
    if screen == "trimmed_mean":
        c["b"] = b
    return dict(c, **kw)


def _setup(graph_key, dtype, attack, screen="trimmed_mean", b=1, n=13, S=3, seed=0):
    conf = _bconf(screen, b)
    if attack:
        conf["byzantine"] = {"nodes": BYZ[graph_key], "attack": attack, "scale": 3.0, "z": 1.5}
    pr = KernelProblem(GRAPHS[graph_key], n, dtype, S, seed=seed, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    o = Bridge(pr, DEV, conf)
    # the rows published for round 0 differ from theta (as after a resume with an attacker)
    o.pub[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, o, conf


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def _check_mix(pr, o, tp, theta0, pub0, theta1, dt, byz):
    """bridge_mix's rows against the oracle (bound: a few row-dtype roundings of the kept values' magnitude), the
    median of an odd count bit for bit, and the screening guarantee on the kernel's output."""
    npdt = NPDT[pr.dtype]
    u = co.unit_roundoff(npdt)
    W = np.zeros((pr.N, pr.N))
    for i in range(pr.N):
        for j in tp.neighbors_noself[i]:
            W[i, j] = 1.0
    for i in range(pr.N):
        nb = list(tp.neighbors_noself[i])
        want = bo.screen(theta0[i], pub0[nb], o.screen, o.b)
        mag = (np.abs(theta0[i]) + np.abs(pub0[nb]).sum(0)) if nb else np.abs(theta0[i])
        _ratio(f"bridge_mix {o.screen}", dt, theta1[i], want, C * u * (np.abs(want) + mag * U64 / u) + 1e-300)
        if o.screen == "median" and len(nb) % 2 == 0:
            assert np.array_equal(theta1[i].astype(npdt).view(np.uint8), want.astype(npdt).view(np.uint8)), \
                f"node {i}: the median of an odd count is not the selected value"
        if bo.guaranteed(W, i, byz, o.screen, o.b):
            lo, hi = bo.honest_range(theta0, pub0, W, i, byz)
            slack = 4 * U64 * (np.abs(lo) + np.abs(hi))
            assert np.all(theta1[i] >= lo - slack) and np.all(theta1[i] <= hi + slack), f"node {i}: outside the range"


def _run_checked(pr, o, eng, rounds=ROUNDS):
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    u = co.unit_roundoff(NPDT[pr.dtype])
    L = pr.N
    op = eng.op
    byz = set(o.byzantine)
    for k in range(rounds):
        par = k & 1
        tp = Topology(pr.plan_graphs(o.oits, 0, 1)[k])
        theta0, pub0 = _t(pr.arena.theta), _t(eng.pub[par, 0, :L])
        op.bridge_mix()
        torch.cuda.synchronize()
        _check_mix(pr, o, tp, theta0, pub0, _t(pr.arena.theta), dt, byz)
        # ---- gradient, then the step; the same state through dsgd_step for the bitwise comparison
        pr.fused.launch()
        torch.cuda.synchronize()
        keep = (pr.arena.theta.clone(), eng.pub.clone(), eng.round_ctr.clone(), pr.fused.calls.clone())
        op.dsgd_step()
        torch.cuda.synchronize()
        ref_theta, ref_pub = pr.arena.theta.clone(), eng.pub[par ^ 1, 0, :L].clone()
        pr.arena.theta.copy_(keep[0]); eng.pub.copy_(keep[1]); eng.round_ctr.copy_(keep[2]); pr.fused.calls.copy_(keep[3])
        op.cg_step()
        torch.cuda.synchronize()
        assert int(eng.round_ctr.item()) == k + 1 and int(eng.done_ctr.item()) == 0
        assert torch.equal(pr.arena.theta, ref_theta), f"round {k}: cg_step theta != dsgd_step theta"
        pub1 = eng.pub[par ^ 1, 0, :L]
        s = torch.tensor(o.scale, dtype=pr.dtype)
        for i in range(L):
            if o.attack[i] == 0:
                assert torch.equal(pub1[i], ref_pub[i]), f"round {k} node {i}: honest row"
            elif o.attack[i] == 1:
                assert torch.equal(pub1[i], -(s * pr.arena.theta[i])), f"round {k} node {i}: sign-flip row"
            else:
                hon = [j for j in tp.neighbors_noself[i] if j not in byz]
                got = _t(pub1[i])
                if not hon:
                    assert np.array_equal(got, _t(pr.arena.theta[i]))
                    continue
                x = pub0[hon]
                want = x.mean(0) - o.z * x.std(0)
                err = 2 * u * np.abs(want) + C * len(hon) * U64 * (np.abs(x).max(0) * (1 + abs(o.z)))
                _ratio("cg_step alie", dt, got, want, err + 1e-300)
        assert not _t(eng.pub[par ^ 1, 0, :L])[:, pr.n:].any() and not _t(pr.arena.theta)[:, pr.n:].any()
    eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("attack", [None, "sign_flip", "alie"])
@pytest.mark.parametrize("screen", ["trimmed_mean", "median"])
@pytest.mark.parametrize("graph_key", sorted(GRAPHS))
def test_launches_match_oracle(graph_key, screen, attack, dtype):
    """Degrees 0 to 9 (isolated, star8, wheel10, random5to7), the complete graph through the pointer table in both of
    its configurations, a graph that changes every round; rows of 13 parameters (padding in the row); b rotates over
    0 .. 3 with the graph."""
    i = sorted(GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, attack, screen, b=i % 4, S=(1, 3, 5, 17)[i % 4], seed=i)
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert not eng.sum_mode and eng.C == 1
    _run_checked(pr, o, eng)


@DTYPES
@pytest.mark.parametrize("b", [0, 1, 2, 3])
def test_every_trim_depth_on_the_wheel(b, dtype):
    """The wheel's hub has 9 neighbors (the 16-slot variant), its rim nodes 3: every b from 0 to 3 keeps some and, at
    b >= 2, leaves a rim node its own row."""
    pr, o, conf = _setup("wheel10", dtype, "alie", "trimmed_mean", b=b, seed=20 + b)
    _run_checked(pr, o, ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1)))


@DTYPES
@pytest.mark.parametrize("screen", ["trimmed_mean", "median"])
@pytest.mark.parametrize("graph_key", ["cycle6", "wheel10"])
def test_grid_stride_rows_match_oracle(graph_key, screen, dtype):
    """Rows long enough that every CTA of a node loops over several vectors."""
    pr, o, conf = _setup(graph_key, dtype, "sign_flip", screen, b=1, n=150_001, S=4, seed=11)
    _run_checked(pr, o, ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1)), rounds=2)


def _permute_tables(eng, perm_of):
    """Reorder each node's neighbor slots (pointer, weight, rank and Byzantine tables) by ``perm_of(l, deg)``."""
    for gi in range(eng.t_deg.shape[0]):
        for l in range(eng.t_deg.shape[1]):
            d = int(eng.t_deg[gi, l])
            p = torch.as_tensor(perm_of(l, d), device=DEV, dtype=torch.long)
            for t in (eng.t_nbr_ptr, eng.t_nbr_w, eng.t_nbr_rank, eng.t_nbr_byz):
                t[gi, l, :d] = t[gi, l, :d][p].clone()


@DTYPES
@pytest.mark.parametrize("screen,b", [("trimmed_mean", 0), ("trimmed_mean", 2), ("median", 0)])
def test_permuted_neighbor_table_gives_the_same_rows(screen, b, dtype):
    """The sorted values do not depend on the table order, so neither do the rows (torch.equal: +0 and -0 compare
    equal).  Rows with ties and zeros between neighbors."""
    pr, o, conf = _setup("wheel10", dtype, "alie", screen, b=b, n=4099, seed=4)
    pub = o.pub
    pub[3, :64] = pub[4, :64]                 # exact ties between neighbors
    pub[2, 64:96] = 0.0
    pub[6, 64:96] = -0.0
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    theta0 = pr.arena.theta.clone()
    eng.op.bridge_mix()
    torch.cuda.synchronize()
    want = pr.arena.theta.clone()
    rng = np.random.default_rng(0)
    _permute_tables(eng, lambda l, d: rng.permutation(d))
    pr.arena.theta.copy_(theta0)
    eng.op.bridge_mix()
    torch.cuda.synchronize()
    assert torch.equal(pr.arena.theta, want)


@pytest.mark.parametrize("screen", ["trimmed_mean", "median"])
def test_permuted_node_order_is_bitwise_the_identity_order(screen):
    """The node order of a multi-GPU launch (nodes with remote neighbors first) only permutes blockIdx.y."""
    outs = []
    for perm in (None, [5, 3, 1, 0, 2, 4]):
        pr, o, conf = _setup("cycle6", torch.float32, "alie", screen, b=1, n=4099, seed=3)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        if perm is not None:
            order = torch.tensor(perm, dtype=torch.int32, device=DEV)
            eng._keep["node_order"] = order.data_ptr()
            eng.op = type(eng.op)(eng._keep)
        for k in range(3):
            eng.op.bridge_mix(); pr.fused.launch(); eng.op.cg_step()
        torch.cuda.synchronize()
        outs.append((pr.arena.theta.clone(), eng.pub.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@DTYPES
@pytest.mark.parametrize("screen,b", [("trimmed_mean", 1), ("median", 0)])
def test_slot_variants_give_the_same_bits(screen, b, dtype):
    """The six nodes of a cycle alone (4 slots), beside a star of degree 6 (8 slots) and beside one of degree 12
    (16 slots): the cycle's rows are bitwise the same, since the slots past deg hold +inf and sort last."""
    outs, slots = [], []
    for hub in (0, 6, 12):
        g = nx.cycle_graph(6)                    # the first six nodes keep cycle_graph(6)'s neighbor order
        if hub:
            g.add_edges_from((6, 7 + j) for j in range(hub))
        GRAPHS["_slots"] = [g]
        try:
            pr, o, conf = _setup("_slots", dtype, None, screen, b=b, n=1025, seed=5)
        finally:
            del GRAPHS["_slots"]
        gen = torch.Generator().manual_seed(9)
        th = torch.randn(6, pr.n, generator=gen, dtype=torch.float64).to(dtype).to(DEV)
        pr.arena.theta[:6, :pr.n] = th
        o.pub[:6, :pr.n] = th + torch.randn(6, pr.n, generator=gen, dtype=torch.float64).to(dtype).to(DEV)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        eng.op.bridge_mix()
        torch.cuda.synchronize()
        outs.append(pr.arena.theta[:6].clone())
        slots.append(eng.dmax)
    assert slots == [2, 6, 12]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


# ------------------------------------------------------------------------------------------- whole runs ----
BR = {"alg_name": "bridge", "alpha0": 0.01, "mu": 0.001, "screen": "trimmed_mean", "b": 1, "outer_iterations": 7,
      "profile": False}
SCREENS = {"trimmed_mean": {"screen": "trimmed_mean", "b": 1}, "median": {"screen": "median"}}
ATTACKS = {"none": None, "sign_flip": {"nodes": [0, 2], "attack": "sign_flip", "scale": 2.0},
           "alie": {"nodes": [0, 1], "attack": "alie", "z": 1.0}}


def _conf(screen="trimmed_mean", **kw):
    c = {k: v for k, v in BR.items() if k != "b"}
    return dict(c, **SCREENS[screen], **kw)


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("screen", sorted(SCREENS))
@pytest.mark.parametrize("attack", sorted(ATTACKS))
def test_mnist_fp64_matches_torch_fp64(attack, screen):
    from test_gpu_mnist import _generic_problem
    conf = _conf(screen)
    if ATTACKS[attack]:
        conf["byzantine"] = ATTACKS[attack]
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b.arena.theta.copy_(a.arena.theta)
    oa = Bridge(a, DEV, copy.deepcopy(conf))
    ob = Bridge(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    ob.pub.copy_(b.arena.theta)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r, rp = _rel(a.arena.theta, b.arena.theta), _rel(oa.pub, ob.pub)
    print(f"\nMNIST fp64 {attack} {screen}: rel theta {r:.2e}, published rows {rp:.2e}")
    assert r < 1e-8 and rp < 1e-8
    staging = 1 if oa._program.host_mode else 0
    assert oa._program.launches_per_round() == staging + 3


def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    conf = _conf("median", byzantine=ATTACKS["alie"])
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = Bridge(pr, DEV, copy.deepcopy(conf))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.pub.clone()))
    for run in outs[1:]:
        for x, y in zip(run, outs[0]):
            assert torch.equal(x, y)


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = _conf("trimmed_mean", outer_iterations=12, byzantine=ATTACKS["sign_flip"])
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = Bridge(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        opt._program.sync_back()
        outs.append((pr.arena.theta.clone(), opt.pub.clone(), pr.forward_cnt))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][2] == outs[1][2]


def test_fused_checkpoint_resume_with_an_alie_attacker_is_bit_exact(tmp_path):
    from test_gpu_mnist import _problem
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf("trimmed_mean", outer_iterations=6, byzantine=ATTACKS["alie"])

    def make():
        return _problem(4, 32, "fused", conf, M=100)
    full = make()
    of = Bridge(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = Bridge(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    second = make()
    o2 = Bridge(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3 and not torch.equal(o2.pub[1], second.arena.theta[1])
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.pub, of.pub)


def test_sequence_check_passes_with_an_alie_attacker_on_a_link_drop_run():
    """The ALIE step reads its honest neighbors' rows of round k after the mix: with ``debug_sequence_check`` and link
    drops every round no stale row is read, and the result matches the PyTorch ops on the same graph sequence."""
    from test_gpu_mnist import _assert_mostly_close, _problem
    outs = []
    for backend in ("fused", "torch"):
        conf = _conf("median", byzantine={"nodes": [0, 3], "attack": "alie", "z": 1.0})
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 7}
        pr._init_faults()
        c = dict(copy.deepcopy(conf), debug_sequence_check=True,
                 consensus_backend="auto" if backend == "fused" else "torch")
        opt = Bridge(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
