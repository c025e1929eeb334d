"""ClippedGossip on the fused sm_90a kernels: ``cg_dist_kernel``, ``cg_mix_kernel`` and ``cg_step_kernel`` one launch at
a time against the float64 rules of ``tests/clipped_gossip_oracle.py`` (fp32 and fp64, degrees 0 to 9, padded and
grid-stride rows, a permuted node order), then whole runs: ``clip: none`` without attackers bitwise fused DSGD, fp64
MNIST under each attack against the PyTorch path, determinism, graph replay, the input pipelines, resume and the
sequence check with an ALIE attacker."""
import collections
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import clipped_gossip_oracle as cgo
import consensus_oracle as co
from test_gpu_consensus_kernels import GRAPHS, KernelProblem
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.optimizers import DSGD, ClippedGossip
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16                      # bound multiplier, as tests/consensus_oracle.py
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
WORST = collections.defaultdict(float)
ROUNDS = 4
# Byzantine nodes per graph: adjacent attackers, an honest node whose only neighbors attack (isolated: 4-5), an
# isolated attacker (6), the hub of the star and the wheel
BYZ = {"path2_ptr": [1], "cycle6": [0, 1], "star8": [0], "wheel10": [0, 5], "random5to7": [2],
       "isolated": [4, 6], "complete6_sum": [0, 1], "complete6_ptr": [0, 1], "switch": [1]}
U64 = 2.0 ** -53


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / bound per launch and dtype:")
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:18s} {dt:5s} {r:.3f}")


def _ratio(name, dt, got, want, err):
    r = float(np.max(np.abs(got - want) / err)) if got.size else 0.0
    WORST[(name, dt)] = max(WORST[(name, dt)], r)
    assert r <= 1.0, f"{name}: worst ratio {r:.3f}"


def _setup(graph_key, dtype, attack, n=13, S=3, delta=0.3, seed=0, clip="adaptive"):
    conf = {"alg_name": "clipped_gossip", "alpha0": 0.08, "mu": 0.5, "clip": clip, "delta": delta,
            "outer_iterations": ROUNDS, "profile": False}
    if attack:
        conf["byzantine"] = {"nodes": BYZ[graph_key], "attack": attack, "scale": 3.0, "z": 1.5}
    pr = KernelProblem(GRAPHS[graph_key], n, dtype, S, seed=seed, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    o = ClippedGossip(pr, DEV, conf)
    # the rows published for round 0 differ from theta (as after a resume with an attacker)
    o.pub[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    return pr, o, conf


def _t(x):
    return x.detach().double().cpu().numpy().copy()


def _run_checked(pr, o, eng, rounds=ROUNDS):
    dt = "fp32" if pr.dtype == torch.float32 else "fp64"
    u = co.unit_roundoff(NPDT[pr.dtype])
    L, n_pad, dmax = pr.N, pr.layout.n_pad, eng.dmax
    op = eng.op
    byz = set(o.byzantine)
    alpha = _t(eng.alpha)
    W_t = _t(eng.t_nbr_w)
    for k in range(rounds):
        par = k & 1
        tp = Topology(pr.plan_graphs(o.oits, 0, 1)[k])
        gid = int(eng.t_gid[k].item())
        theta0, pub0 = _t(pr.arena.theta), _t(eng.pub[par, 0, :L])
        # ---- distances
        op.cg_dist()
        torch.cuda.synchronize()
        parts = eng.dist_part.view(L, dmax, -1).double().cpu().numpy()
        dist = np.sqrt(parts.sum(2))
        for i in range(L):
            nb = tp.neighbors_noself[i]
            want = np.array([np.linalg.norm(pub0[j] - theta0[i]) for j in nb])
            _ratio("cg_dist", dt, dist[i, :len(nb)], want, C * n_pad * U64 * np.maximum(want, 1e-300) + 1e-300)
        # ---- mix, with the radius decided from the kernel's distances
        op.cg_mix()
        torch.cuda.synchronize()
        theta1 = _t(pr.arena.theta)
        for i in range(L):
            nb = tp.neighbors_noself[i]
            w = W_t[gid, i, :len(nb)]
            f, _, _ = cgo.radius(dist[i, :len(nb)], w, o.delta)
            coef = np.array([NPDT[pr.dtype](w[e] * f[e]) for e in range(len(nb))], dtype=np.float64)
            want = theta0[i] + sum(coef[e] * (pub0[j] - theta0[i]) for e, j in enumerate(nb))
            err = np.abs(theta0[i]) + sum(abs(coef[e]) * (np.abs(pub0[j]) + np.abs(theta0[i])) for e, j in enumerate(nb))
            _ratio("cg_mix", dt, theta1[i], want, C * u * (err + 1e-300) + 1e-300)
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
                mu, sg = x.mean(0), x.std(0)
                want = mu - o.z * sg
                err = 2 * u * np.abs(want) + C * len(hon) * U64 * (np.abs(x).max(0) * (1 + abs(o.z)))
                _ratio("cg_step alie", dt, got, want, err + 1e-300)
        assert not _t(eng.pub[par ^ 1, 0, :L])[:, pr.n:].any() and not _t(pr.arena.theta)[:, pr.n:].any()
    eng.check()


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("attack", [None, "sign_flip", "alie"])
@pytest.mark.parametrize("graph_key", sorted(GRAPHS))
def test_launches_match_oracle(graph_key, attack, dtype):
    """Degrees 0 to 9 (isolated, star8, wheel10, random5to7), the complete graph through the pointer table in both of
    its configurations, a graph that changes every round; rows of 13 parameters (padding in the row)."""
    i = sorted(GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, attack, S=(1, 3, 5, 17)[i % 4], delta=(0.0, 0.2, 0.3, 0.45)[i % 4], seed=i)
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    assert not eng.sum_mode and eng.C == 1
    _run_checked(pr, o, eng)


@DTYPES
@pytest.mark.parametrize("attack", ["sign_flip", "alie"])
def test_grid_stride_rows_match_oracle(attack, dtype):
    """Rows long enough that every CTA of a node loops over several vectors and cg_mix sums many partials."""
    pr, o, conf = _setup("cycle6", dtype, attack, n=150_001, S=4, seed=11)
    eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
    _run_checked(pr, o, eng, rounds=2)
    per_block = 256 * (4 if dtype == torch.float32 else 2)
    assert eng.dist_part.numel() // (pr.N * eng.dmax) == -(-pr.layout.n_pad // per_block)


@DTYPES
def test_distances_do_not_depend_on_the_grid(dtype):
    """Six nodes alone and beside six more (two disjoint cycles): with rows this long the one-wave grid of the twelve
    nodes has fewer CTAs per node, yet the distance partials are per chunk of the row, so the first six nodes' rows
    are bitwise those of the six alone (what makes a multi-rank run equal a single-process one)."""
    twin = nx.cycle_graph(6)
    nx.add_cycle(twin, range(6, 12))          # the first six nodes keep cycle_graph(6)'s neighbor order
    outs = []
    for graph in (nx.cycle_graph(6), twin):
        GRAPHS["_grid"] = [graph]
        try:
            pr, o, conf = _setup("_grid", dtype, None, n=150_001, S=4, seed=5)
        finally:
            del GRAPHS["_grid"]
        g = torch.Generator().manual_seed(9)
        th = torch.randn(6, pr.n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        pr.arena.theta[:, :pr.n] = th.repeat(pr.N // 6, 1)
        o.pub[:, :pr.n] = (th + 0.1 * torch.randn(6, pr.n, generator=g, dtype=torch.float64).to(dtype).to(DEV)).repeat(pr.N // 6, 1)
        # the same gradients for both copies (the first six rows of base are drawn alike for any node count)
        pr.fused.base.copy_(pr.fused.base[:6].repeat(pr.N // 6, 1, 1))
        pr.fused.slope.zero_()
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        for k in range(3):
            eng.op.cg_dist(); eng.op.cg_mix(); pr.fused.launch(); eng.op.cg_step()
        torch.cuda.synchronize()
        outs.append(pr.arena.theta[:6].clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("attack", [None, "alie"])
def test_permuted_node_order_is_bitwise_the_identity_order(attack):
    """The node order of a multi-GPU launch (nodes with remote neighbors first) only permutes blockIdx.y."""
    outs = []
    for perm in (None, [5, 3, 1, 0, 2, 4]):
        pr, o, conf = _setup("cycle6", torch.float32, attack, n=4099, seed=3)
        eng = ConsensusEngine(o, pr.plan_graphs(o.oits, 0, 1))
        if perm is not None:
            order = torch.tensor(perm, dtype=torch.int32, device=DEV)
            eng._keep["node_order"] = order.data_ptr()
            eng.op = type(eng.op)(eng._keep)
        for k in range(3):
            eng.op.cg_dist(); eng.op.cg_mix(); pr.fused.launch(); eng.op.cg_step()
        torch.cuda.synchronize()
        outs.append((pr.arena.theta.clone(), eng.pub.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


# ------------------------------------------------------------------------------------------- whole runs ----
CG = {"alg_name": "clipped_gossip", "alpha0": 0.01, "mu": 0.001, "clip": "adaptive", "delta": 0.2,
      "outer_iterations": 7, "profile": False}
ATTACKS = {"none": None, "sign_flip": {"nodes": [0, 2], "attack": "sign_flip", "scale": 2.0},
           "alie": {"nodes": [0, 1], "attack": "alie", "z": 1.0}}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("graph", ["cycle", "complete"])
def test_clip_none_without_attackers_is_fused_dsgd_bitwise(graph):
    from test_gpu_mnist import _problem
    g = nx.cycle_graph(5) if graph == "cycle" else nx.complete_graph(5)
    outs, launches = [], []
    for conf in (dict(CG, clip="none"), {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 7,
                                         "profile": False}):
        conf["complete_graph_mode"] = "pointer"
        pr = _problem(5, 32, "fused", conf, graph=g, eval_every=3)
        opt = (ClippedGossip if conf["alg_name"] == "clipped_gossip" else DSGD)(pr, DEV, copy.deepcopy(conf))
        opt.train()
        launches.append(opt._program.launches_per_round())
        outs.append(pr.arena.theta.clone())
    assert torch.equal(outs[0], outs[1])
    assert launches[0] == launches[1]


@pytest.mark.parametrize("clip", ["none", "adaptive"])
@pytest.mark.parametrize("attack", sorted(ATTACKS))
def test_mnist_fp64_matches_torch_fp64(attack, clip):
    from test_gpu_mnist import _generic_problem
    conf = dict(CG, clip=clip)
    if ATTACKS[attack]:
        conf["byzantine"] = ATTACKS[attack]
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b.arena.theta.copy_(a.arena.theta)
    oa = ClippedGossip(a, DEV, copy.deepcopy(conf))
    ob = ClippedGossip(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    ob.pub.copy_(b.arena.theta)
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    r, rp = _rel(a.arena.theta, b.arena.theta), _rel(oa.pub, ob.pub)
    print(f"\nMNIST fp64 {attack} clip={clip}: rel theta {r:.2e}, published rows {rp:.2e}")
    assert r < 1e-8 and rp < 1e-8
    staging = 1 if oa._program.host_mode else 0
    assert oa._program.launches_per_round() == staging + (4 if clip == "adaptive" else 3)


def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    conf = dict(CG, byzantine=ATTACKS["alie"])
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=3)
        opt = ClippedGossip(pr, DEV, copy.deepcopy(conf))
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
        conf = dict(CG, outer_iterations=12, byzantine=ATTACKS["sign_flip"])
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = ClippedGossip(pr, DEV, conf)
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
    conf = dict(CG, outer_iterations=6, byzantine=ATTACKS["alie"])

    def make():
        return _problem(4, 32, "fused", conf, M=100)
    full = make()
    of = ClippedGossip(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = ClippedGossip(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    second = make()
    o2 = ClippedGossip(second, DEV, copy.deepcopy(conf))
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
        conf = dict(CG, byzantine={"nodes": [0, 3], "attack": "alie", "z": 1.0})
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 7}
        pr._init_faults()
        c = dict(copy.deepcopy(conf), debug_sequence_check=True,
                 consensus_backend="auto" if backend == "fused" else "torch")
        opt = ClippedGossip(pr, DEV, c)
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])
