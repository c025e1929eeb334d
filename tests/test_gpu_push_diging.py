"""Push-DIGing on the fused sm_90a kernels: ``pdg_mix`` and ``pdg_track`` one launch at a time against a float64
oracle (|kernel - oracle| <= 16 u err), theta bitwise u / w with the stored w and the published rows bitwise the
kernel's own, then whole runs against the PyTorch path, determinism, CUDA-graph replay, the input pipelines,
checkpoint/resume and the sequence check."""
import collections
import copy

import numpy as np
import pytest
import torch

import consensus_oracle as co
from test_gpu_consensus_kernels import KernelProblem
from test_gpu_sgp import SGP_GRAPHS, _density64, _gen, _mnist64, _rdg, _rel
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.ops.engine import ConsensusEngine
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import PushDIGing
from nn_distributed_training_b200.utils.graph_generation import Topology

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 16
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
WORST = collections.defaultdict(float)
ROUNDS, CHECKED = 6, (0, 1, 5)
S_LIST = [1, 3, 4, 5, 16, 17]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) per kernel and dtype (c = %d):" % C)
    for (kern, dt), r in sorted(WORST.items()):
        print(f"  {kern:10s} {dt:5s} {r:.3f}")


# ------------------------------------------------------------------------------------------------ harness ----
def _setup(graph_key, dtype, S, n, n_pad=None, seed=0, oits=ROUNDS):
    """Push-sum weights far from 1 with theta = u / w, and nonzero trackers and previous gradients, so every term of
    both kernels is live from round 0."""
    conf = {"alg_name": "push_diging", "alpha": 0.07, "outer_iterations": oits, "profile": False}
    pr = KernelProblem(SGP_GRAPHS[graph_key], n, dtype, S, seed=seed, n_pad=n_pad, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    th = torch.randn(pr.N, n, generator=g, dtype=torch.float64)
    pr.arena.theta[:, :n] = th.to(dtype).to(DEV)
    o = PushDIGing(pr, DEV, conf)
    o.w.copy_(torch.exp(2.0 * torch.randn(pr.N, generator=g, dtype=torch.float64)).to(DEV))
    o.u.copy_(pr.arena.theta * o.w.to(dtype).unsqueeze(1))
    pr.arena.theta.copy_(ref.sgp_debias(o.u, o.w))
    o.y[:, :n] = (0.5 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    o.g[:, :n] = (0.5 * torch.randn(pr.N, n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    return pr, o, conf


def _state(pr, o, eng):
    L, n_pad = pr.N, pr.layout.n_pad
    t = lambda x: x.detach().double().cpu().numpy().copy()
    c = lambda x: x.detach().cpu().clone()
    return dict(theta=t(pr.arena.theta), u=t(o.u), w=t(o.w), ysum=t(o.ysum), g_old=t(o.g),
                theta_t=c(pr.arena.theta), u_t=c(o.u), w_t=c(o.w), ysum_t=c(o.ysum), g_old_t=c(o.g),
                pub=t(eng.pub[:, :, :L, :n_pad]), pub_t=c(eng.pub[:, :, :L, :n_pad]),
                pub_w=np.stack([t(eng.pub_weights(p)) for p in (0, 1)]),
                pub_tail=eng.pub[:, 0, :L].view(torch.uint8)[..., n_pad * eng.pub.element_size():].cpu().clone(),
                calls=pr.fused.calls.cpu().numpy().copy(), round_ctr=int(eng.round_ctr.item()),
                done_ctr=int(eng.done_ctr.item()), grad_part=t(pr.fused.grad_part))


class Harness:
    def __init__(self, pr, o):
        self.pr, self.o = pr, o
        self.graphs = pr.plan_graphs(o.oits, 0, 1)
        self.eng = ConsensusEngine(o, self.graphs)
        assert not self.eng.sum_mode and self.eng.C == 2
        assert self.eng.bytes_per_round()["row"] == 2 * (pr.layout.n_pad * o.u.element_size() + 16)
        self.npdt = NPDT[pr.dtype]
        self.u = co.unit_roundoff(self.npdt)
        self.dt = "fp32" if pr.dtype == torch.float32 else "fp64"
        self.alpha = self.eng.alpha.cpu().double().numpy()
        self.n = pr.n

    def launch(self, name, fn, k, check=True):
        before = _state(self.pr, self.o, self.eng)
        fn()
        torch.cuda.synchronize()
        after = _state(self.pr, self.o, self.eng)
        if name == "grad":
            return
        par, n, u = k & 1, self.n, self.u
        assert after["done_ctr"] == 0, name
        ends = name == "pdg_track"
        assert after["round_ctr"] == before["round_ctr"] + (1 if ends else 0), name
        assert np.array_equal(after["calls"], before["calls"] + (1 if ends else 0)), name
        for key in ("theta", "u", "ysum", "g_old"):
            assert not after[key][:, n:].any(), f"{name}: padding of {key} written"
        # every element of theta is u / w with the stored w: all CTAs of a node divided by the same bits
        assert torch.equal(after["theta_t"], ref.sgp_debias(after["u_t"], after["w_t"])), f"{name} round {k}: theta != u / w"
        key = (name, self.dt)
        if name == "pdg_mix":
            assert torch.equal(after["pub_t"], before["pub_t"]) and torch.equal(after["pub_tail"], before["pub_tail"])
            assert torch.equal(after["g_old_t"], before["g_old_t"])
            if not check:
                return
            tp = Topology(self.graphs[k])
            A = tp.push_weights.astype(self.npdt).astype(np.float64)      # the kernel's weights
            nbrs = tp.neighbors_noself
            us, ys, ws = before["pub"][par, 0], before["pub"][par, 1], before["pub_w"][par]
            a = self.alpha[k]
            x, e_x = np.zeros_like(us), np.zeros_like(us)
            s, e_s = np.zeros_like(us), np.zeros_like(us)
            w, e_w = np.zeros(self.pr.N), np.zeros(self.pr.N)
            for i in range(self.pr.N):
                own = before["u"][i] - a * ys[i]
                x[i] = A[i, i] * own
                mag = A[i, i] * (np.abs(before["u"][i]) + a * np.abs(ys[i]))
                for j in nbrs[i]:
                    x[i] += A[i, j] * (us[j] - a * ys[j])
                    mag += A[i, j] * (np.abs(us[j]) + a * np.abs(ys[j]))
                e_x[i] = u * (2.0 * mag + np.abs(x[i]))
                s[i], e_s[i] = co._mix(i, ys[i], ys, nbrs, A, u)
                wi, wm = A[i, i] * ws[i], abs(A[i, i] * ws[i])
                for j in nbrs[i]:
                    wi += A[i, j] * ws[j]
                    wm += abs(A[i, j] * ws[j])
                w[i], e_w[i] = wi, co.U64 * (wm + abs(wi))
            th = x / w[:, None]
            e_th = (e_x + np.abs(th) * e_w[:, None]) / w[:, None] + 2 * u * np.abs(th)
            WORST[key] = max(WORST[key], co.check(f"{name} round {k} w", after["w"], w, e_w, C),
                             co.check(f"{name} round {k} u", after["u"], x, e_x, C),
                             co.check(f"{name} round {k} ysum", after["ysum"], s, e_s, C),
                             co.check(f"{name} round {k} theta", after["theta"], th, e_th, C))
            return
        # pdg_track: reads only local rows, writes g_old and the other parity
        for name_t in ("w_t", "u_t", "ysum_t", "theta_t"):
            assert torch.equal(after[name_t], before[name_t]), f"pdg_track wrote {name_t}"
        assert torch.equal(after["pub_t"][par], before["pub_t"][par]), "pdg_track wrote the parity being read"
        assert torch.equal(after["pub_tail"][par], before["pub_tail"][par])
        assert torch.equal(after["pub_t"][par ^ 1, 0], after["u_t"]), f"{name} round {k}: published u"
        assert np.array_equal(after["pub_w"][par ^ 1], after["w"]), f"{name} round {k}: published w"
        # the published tracker is the kernel's y = ysum + (g - g_old), in the kernel's dtype
        y_own = before["ysum_t"] + (after["g_old_t"] - before["g_old_t"])
        assert torch.equal(after["pub_t"][par ^ 1, 1], y_own), f"{name} round {k}: published y"
        if not check:
            return
        g, e_g = co.sum_partials(before["grad_part"], u)
        yn = before["ysum"] + g - before["g_old"]
        e_y = e_g + u * (np.abs(before["ysum"]) + np.abs(g) + np.abs(before["g_old"]) + np.abs(yn))
        WORST[key] = max(WORST[key], co.check(f"{name} round {k} g_old", after["g_old"], g, e_g, C),
                         co.check(f"{name} round {k} y", after["pub"][par ^ 1, 1], yn, e_y, C))

    def run(self, rounds=ROUNDS, checked=CHECKED):
        op, src = self.eng.op, self.pr.fused
        for k in range(rounds):
            chk = k in checked
            self.launch("pdg_mix", op.pdg_mix, k, check=chk)
            self.launch("grad", src.launch, k)
            self.launch("pdg_track", op.pdg_track, k, check=chk)
        self.eng.check()


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


# ------------------------------------------------------------------------------------------ per launch ----
@DTYPES
@pytest.mark.parametrize("graph_key", sorted(SGP_GRAPHS))
def test_launches_match_oracle(graph_key, dtype):
    """In-degrees 0-9 (a node with no in-neighbors and six readers among them), undirected and directed graphs, a graph
    that changes every round, rows of 77 parameters padded to the row alignment, S rotating with the case."""
    i = sorted(SGP_GRAPHS).index(graph_key)
    pr, o, conf = _setup(graph_key, dtype, S_LIST[i % len(S_LIST)], n=77, seed=i)
    Harness(pr, o).run()


@DTYPES
@pytest.mark.parametrize("S", S_LIST)
def test_every_partial_count_matches_oracle(S, dtype):
    """The 4-deep and 8-deep partial sums and the tail loop past 8 (degree-9 hub: both neighbor groups)."""
    pr, o, conf = _setup("wheel10", dtype, S, n=100, seed=S)
    Harness(pr, o).run(rounds=2, checked=(0, 1))


@DTYPES
@pytest.mark.parametrize("size", ["one_unit", "grid_stride"])
def test_row_sizes_match_oracle(size, dtype):
    """A row shorter than a CTA's span, and rows long enough that the grid is capped at the resident CTAs and every
    node has many CTAs, all of which must agree on w."""
    if size == "one_unit":
        pr, o, conf = _setup("random_directed", dtype, 5, n=128, seed=3)
        Harness(pr, o).run()
        return
    pr, o, conf = _setup("exponential10", dtype, 17, n=140001, seed=4)
    Harness(pr, o).run(rounds=2, checked=(0, 1))


@DTYPES
def test_graph_replay_equals_eager_launches(dtype):
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup("switch", dtype, 5, n=300, seed=2)
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
PD = {"alg_name": "push_diging", "alpha": 0.05, "outer_iterations": 7, "profile": False}


def _compare(tag, fused, torch_path, of, ot):
    for name, x, y in (("theta", fused.arena.theta, torch_path.arena.theta), ("u", of.u, ot.u), ("w", of.w, ot.w)):
        r = _rel(x, y)
        print(f"{tag} {name}: rel {r:.2e}")
        assert r < 1e-13, name
    # the tracker is a sum of gradient differences: its rounding is measured against the size of the gradients
    r = ((of.y - ot.y).norm() / ot.g.norm()).item()
    print(f"{tag} y: rel to |g| {r:.2e}")
    assert r < 1e-12, "y"


@pytest.mark.parametrize("model", ["mnist_paper_fp64", "density_fp64"])
def test_fp64_runs_match_torch_path(model):
    make = _mnist64 if model == "mnist_paper_fp64" else _density64
    a, b = make(PD, "fused"), make(PD, "torch")
    b.arena.theta.copy_(a.arena.theta)
    oa = PushDIGing(a, DEV, copy.deepcopy(PD))
    ob = PushDIGing(b, DEV, dict(copy.deepcopy(PD), consensus_backend="torch"))
    assert oa._use_engine() and not ob._use_engine()
    oa.train()
    ob.train()
    assert (oa.w - 1.0).abs().max() > 1e-2
    assert torch.isfinite(a.arena.theta).all()
    _compare(model, a, b, oa, ob)
    assert a.forward_cnt == b.forward_cnt


def test_online_density_fp64_dynamic_graph_matches_torch_fp64(tmp_path):
    """The online problem (graph planned from the robot poses, changing over the run) in float64."""
    from test_gpu_mlp_f64 import _online_problem
    oc = dict(PD, alpha=0.002, outer_iterations=9)
    fused = _online_problem("fused", str(tmp_path), oc)
    refp = _online_problem("torch", str(tmp_path), oc)
    refp.arena.theta.copy_(fused.arena.theta)
    of = PushDIGing(fused, DEV, copy.deepcopy(oc))
    orf = PushDIGing(refp, DEV, dict(copy.deepcopy(oc), consensus_backend="torch"))
    orf.train()
    of.train()
    assert len(of._program.eng.topos) > 1
    assert (fused.positions() == refp.positions()).all()
    assert fused.forward_cnt == refp.forward_cnt
    for key in ("validation_loss", "train_loss_moving_average"):
        torch.testing.assert_close(fused.metrics[key][-1], refp.metrics[key][-1], rtol=1e-9, atol=1e-12)
    _compare("online density", fused, refp, of, orf)


# ------------------------------------------------------------------------- determinism and resume ----
def test_runs_are_deterministic_and_graph_replay_equals_no_graph(monkeypatch):
    from test_gpu_mnist import _problem
    outs = []
    for no_graph in ("0", "0", "1"):
        monkeypatch.setenv("NNDT_NO_GRAPH", no_graph)
        pr = _problem(5, 32, "fused", copy.deepcopy(PD), graph=_gen("exponential", 5), eval_every=3)
        opt = PushDIGing(pr, DEV, copy.deepcopy(PD))
        opt.train()
        assert opt._program.capturable == (no_graph == "0")
        outs.append((pr.arena.theta.clone(), opt.u.clone(), opt.w.clone(), opt.y.clone(), opt.g.clone()))
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0]))


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_mnist_input_pipelines_match_resident(pipeline):
    from test_gpu_mnist import _problem
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(PD, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, graph=_rdg(4), eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = PushDIGing(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        opt._program.sync_back()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), opt.u.clone(), opt.w.clone(), opt.y.clone(), pr.forward_cnt))
        assert torch.isfinite(pr.arena.theta).all() and not torch.all(opt.w == 1.0)
    assert all(torch.equal(x, y) for x, y in zip(outs[0][:4], outs[1][:4]))
    assert outs[0][4] == outs[1][4]


@pytest.mark.parametrize("model", ["mnist_fp32", "density_fp64"])
def test_fused_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, model):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = dict(PD, outer_iterations=6)
    if model == "mnist_fp32":
        from test_gpu_mnist import _problem

        def make():
            return _problem(4, 32, "fused", conf, M=100, graph=_rdg(4))
    else:
        def make():
            return _density64(conf, "fused")
    full = make()
    of = PushDIGing(full, DEV, copy.deepcopy(conf))
    of.train()
    first = make()
    o1 = PushDIGing(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3 and not torch.all(o1.w == 1.0) and o1.y.abs().max() > 0
    second = make()
    o2 = PushDIGing(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    for name in ("u", "w", "y", "g"):
        assert torch.equal(getattr(o2, name), getattr(o1, name)), name
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in ("u", "w", "y", "g"):
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt


def test_sequence_check_passes_on_a_push_diging_run():
    """``debug_sequence_check``: every in-neighbor row read is tagged with the current round."""
    from test_gpu_mnist import _problem
    conf = dict(PD, debug_sequence_check=True, outer_iterations=10)
    pr = _problem(6, 32, "fused", conf, graph=_gen("exponential", 6), eval_every=1000)
    opt = PushDIGing(pr, DEV, conf)
    opt.train()
    assert opt._program.eng.seq_buf is not None
    opt._program.eng.check()
