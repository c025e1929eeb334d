"""The distributed-PPO consensus rounds on the fused sm_90a kernels (``consensus_backend: fused`` / ``--consensus cuda``).

* ``dsgt_mix`` with a per-coordinate step row, with the own-tracker step (theta_i <- sum_j W_ij theta_j - alpha y_i)
  and with both, one launch at a time against the float64 oracle of ``consensus_oracle``: |kernel - oracle| <= 16 u err
  on every coordinate, exact where err = 0.
* Graph replay equals eager launches, bitwise, for those variants and for each trainer's iterations.
* The trainers against the torch consensus path on the recorded batches of ``test_gpu_ppo_update``, in the eager mode
  around per-node autograd, the agreement metric, the non-finite-actor check and the three entry points end to end.
"""
import collections
import os

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
from test_gpu_consensus_kernels import C, NPDT, ROUNDS, Harness, KernelProblem, _snap
from ppo_oracle import F32_FLOOR, rel as _rel
from test_gpu_ppo_update import _batch, _copy_params, _load, _problem
from nn_distributed_training_b200.ops.round_program import RoundProgram
from nn_distributed_training_b200.optimizers import DSGT
from nn_distributed_training_b200.rl import DSGDPPO, DSGTPPO, DiNNOPPO
from nn_distributed_training_b200.rl.consensus_ppo import agreement

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = collections.defaultdict(float)
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |kernel - oracle| / (c err) of dsgt_mix per variant and dtype (c = %d):" % C)
    for (v, dt), r in sorted(WORST.items()):
        print(f"  {v:8s} {dt:5s} {r:.3f}")


# ----------------------------------------------------------------------------------- per-launch oracle ----
def _isolated():
    g = nx.Graph([(0, 1), (1, 2), (2, 3), (3, 0), (0, 2), (4, 5)])
    g.add_node(6)
    return nx.convert_node_labels_to_integers(g)


def _degrees_5_to_7():
    for seed in range(10000):
        g = nx.gnp_random_graph(10, 0.6, seed=seed)
        if min(d for _, d in g.degree()) == 5 and max(d for _, d in g.degree()) == 7:
            return g
    raise AssertionError("no seed gives degrees 5..7")


GRAPHS = {   # name -> (graph, complete_graph_mode)
    "path2_ptr": (nx.path_graph(2), "pointer"),
    "cycle4": (nx.cycle_graph(4), "sum"),
    "star8": (nx.star_graph(8), "sum"),
    "random5to7": (_degrees_5_to_7(), "sum"),
    "isolated": (_isolated(), "sum"),
    "k3_sum": (nx.wheel_graph(3), "sum"),
    "k3_ptr": (nx.wheel_graph(3), "pointer"),
    "k6_sum": (nx.complete_graph(6), "sum"),
    "k6_ptr": (nx.complete_graph(6), "pointer"),
}
VARIANTS = ["row", "own", "row_own"]


def _setup(graph_key, variant, dtype, n=13, S=3, seed=0):
    """A DSGT run of the variant on the test-local gradient source; y starts at the first gradient (dsgt_init) so the
    tracker term is live from round 0.  Coordinates 0, 5, 10 have a zero gradient and a zero step."""
    graph, mode = GRAPHS[graph_key]
    conf = {"alg_name": "dsgt", "alpha": 0.03, "init_grads": True, "outer_iterations": ROUNDS, "profile": False,
            "own_tracker_step": "own" in variant, "complete_graph_mode": mode}
    zero = slice(0, n, 5)
    pr = KernelProblem([graph], n, dtype, S, seed=seed, zero_cols=zero, conf=conf)
    g = torch.Generator().manual_seed(seed + 1)
    pr.arena.theta[:, :n] = torch.randn(pr.N, n, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    pr.arena.theta[:, zero] = 0
    o = DSGT(pr, DEV, conf)
    if "row" in variant:
        row = torch.zeros(pr.arena.n_pad, dtype=torch.float64)
        row[:n] = 0.01 + 0.1 * torch.rand(n, generator=g, dtype=torch.float64)
        row[zero] = 0
        o.alpha = row.to(dtype).to(DEV)
    return pr, o, conf


class VariantHarness(Harness):
    """``Harness`` with the dsgt_mix oracle of the variants: the per-coordinate step broadcasts through
    ``consensus_oracle.dsgt_mix``; the own-tracker step is ``dsgd_mix`` (the mixed theta, or S / N) minus alpha y_i."""

    def __init__(self, pr, o, conf):
        # a per-coordinate step leaves the alpha_k schedule at 0
        super().__init__(pr, o, dict(conf, alpha=0.0) if torch.is_tensor(o.alpha) else conf)

    def _oracle(self, name, k, p, st):
        if name != "dsgt_mix":
            return super()._oracle(name, k, p, st)
        o, eng, u = self.o, self.eng, self.u
        tp = self.topo(k)
        sums = None
        if eng.sum_mode:
            s = st["sum_local"][k & 1]
            sums = (s, co.U64 * np.abs(s))
        kw = dict(k=k, nbrs=tp.neighbors_noself, W=tp.W, u=u, sum_mode=eng.sum_mode, sums=sums)
        alpha = o.alpha.double().cpu().numpy() if torch.is_tensor(o.alpha) else self.alpha[k]
        if not o.own_tracker_step:
            return co.dsgt_mix(st, alpha=alpha, **kw)
        mixed, e_mixed = co.dsgd_mix(st, **kw)
        y = st["pub"][k & 1, 1]                       # node i's own published tracker, not mixed
        th = mixed["theta"] - alpha * y
        return dict(st, theta=th), {"theta": e_mixed["theta"] + u * (np.abs(alpha * y) + np.abs(th))}


@DTYPES
@pytest.mark.parametrize("graph_key", sorted(GRAPHS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_dsgt_mix_variants_match_oracle(variant, graph_key, dtype):
    pr, o, conf = _setup(graph_key, variant, dtype, seed=sorted(GRAPHS).index(graph_key))
    h = VariantHarness(pr, o, conf)
    assert h.eng.sum_mode == (GRAPHS[graph_key][1] == "sum" and nx.density(GRAPHS[graph_key][0]) == 1.0)
    assert (h.eng.alpha_row is not None) == ("row" in variant)
    h.run()
    key = (variant, "fp32" if dtype == torch.float32 else "fp64")
    WORST[key] = max(WORST[key], h.worst["dsgt_mix"])


@DTYPES
@pytest.mark.parametrize("graph_key", ["k3_sum", "cycle4"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_dsgt_variants_graph_replay_equals_eager(variant, graph_key, dtype):
    runs = []
    for capture in (False, True):
        pr, o, conf = _setup(graph_key, variant, dtype, n=300, S=5, seed=2)
        prog = RoundProgram(o)
        prog.capturable = capture
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
            assert np.array_equal(x, b[key]) if isinstance(x, np.ndarray) else x == b[key], f"round {k}: {key}"


# ------------------------------------------------------------------------------------------- trainers ----
DINNO = {"rho_init": 1.0, "rho_scaling": 1.0, "primal_lr_start": 3e-4, "primal_lr_finish": 1e-3,
         "lr_decay_type": "constant", "persistant_primal_opt": False, "primal_iterations": 5, "outer_iterations": 10 ** 6}
TRAINERS = {
    "dinno": (DiNNOPPO, DINNO, False),
    "dsgd": (DSGDPPO, {"alpha0": 3e-3, "mu": 0.0}, False),
    "dsgt": (DSGTPPO, {"alpha_actor": 3e-3, "alpha_critic": 1e-2}, False),      # own-tracker step, per-slot alpha
    "dsgt_init": (DSGTPPO, {"alpha_actor": 3e-3, "alpha_critic": 1e-2, "init_grads": True}, True),
}
PPO_GRAPHS = {"wheel3": (3, None), "cycle4": (4, nx.cycle_graph(4))}


def _params(pr):
    return torch.cat([torch.nn.utils.parameters_to_vector(pr.models[i].parameters()) for i in range(pr.N)])


def _run(name, graph_key, dtype, backend, update="cuda", src=None, batch=None, iters=3):
    """``iters`` iterations on one fixed recorded batch; returns (trainer, final parameters, logged actor losses)."""
    cls, conf, before = TRAINERS[name]
    N, graph = PPO_GRAPHS[graph_key]
    pr = _problem(N, (64, 64, 64), dtype, update_backend=update, n_updates_per_iteration=5)
    if graph is not None:
        pr.graph = graph
    if src is not None:
        _copy_params(pr, src)
    batch = _batch(pr, 800) if batch is None else batch
    tr = cls(pr, DEV, dict(conf, max_rl_timesteps=10 ** 9, writeout=False, consensus_backend=backend))
    start = _params(pr).clone()
    losses = []
    for k in range(iters):
        _load(pr, batch)
        pr.update_advantage()
        if k == 0 and before:
            tr.inner._before_training()
        tr._consensus(k)
        pr.check_update()
        losses += [float(x) for x in pr.logger["actor_losses"]]
        pr.logger["actor_losses"] = []
    out = _params(pr).clone()
    assert torch.isfinite(out).all() and not torch.equal(out, start)
    return tr, out, losses


@pytest.mark.parametrize("graph_key", sorted(PPO_GRAPHS))
@pytest.mark.parametrize("name", sorted(TRAINERS))
def test_trainer_graph_replay_equals_eager(name, graph_key, monkeypatch):
    runs = []
    for eager in (False, True):
        if eager:
            monkeypatch.setenv("NNDT_NO_GRAPH", "1")
        tr, out, losses = _run(name, graph_key, torch.float32, "fused")
        assert tr.inner._program.capturable == (not eager)
        runs.append((out, losses))
    assert torch.equal(runs[0][0], runs[1][0])
    N = PPO_GRAPHS[graph_key][0]
    assert runs[0][1] == runs[1][1] and len(runs[0][1]) == (3 * 5 + TRAINERS[name][2]) * N


@pytest.mark.parametrize("graph_key", sorted(PPO_GRAPHS))
@pytest.mark.parametrize("name", sorted(TRAINERS))
def test_trainer_fp64_matches_torch_consensus(name, graph_key):
    tr, fused, lf = _run(name, graph_key, torch.float64, "fused")
    assert tr.inner._program.eng.sum_mode == (graph_key == "wheel3")
    _, ref, lt = _run(name, graph_key, torch.float64, "torch")
    assert _rel(fused, ref) < 1e-8
    assert np.allclose(lf, lt, rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("graph_key", sorted(PPO_GRAPHS))
@pytest.mark.parametrize("name", sorted(TRAINERS))
def test_trainer_fp32_error_within_4x_of_torch_fp32(name, graph_key):
    N, _ = PPO_GRAPHS[graph_key]
    src = _problem(N, (64, 64, 64), torch.float64)
    batch = {k: v.float() for k, v in _batch(src, 800).items()}     # fp32-representable for all three runs
    _, ref, _ = _run(name, graph_key, torch.float64, "torch", src=src, batch=batch)
    _, t32, _ = _run(name, graph_key, torch.float32, "torch", src=src, batch=batch)
    _, f32, _ = _run(name, graph_key, torch.float32, "fused", src=src, batch=batch)
    e_t, e_f = _rel(t32, ref), _rel(f32, ref)
    print(f"\nfp32 {name} {graph_key}: fused {e_f:.3e} torch {e_t:.3e}")
    assert e_f <= 4 * max(e_t, F32_FLOOR)


@pytest.mark.parametrize("name", sorted(TRAINERS))
def test_eager_mode_with_the_torch_update_matches(name):
    """--consensus cuda --update torch: the consensus kernels eagerly around per-node autograd."""
    tr, fused, lf = _run(name, "wheel3", torch.float64, "fused", update="torch")
    assert not tr.inner._program.capturable
    _, ref, lt = _run(name, "wheel3", torch.float64, "torch", update="torch")
    assert _rel(fused, ref) < 1e-8
    assert np.allclose(lf, lt, rtol=1e-8, atol=1e-12)


@DTYPES
@pytest.mark.parametrize("graph_key", sorted(PPO_GRAPHS))
def test_agreement_metric_kernel_matches_agreement(graph_key, dtype):
    tr, _, _ = _run("dsgt", graph_key, dtype, "fused", iters=2)
    got, want = tr.agreement(), agreement(tr.pr)
    assert got.shape == want.shape == (tr.pr.N,) and got.dtype == want.dtype
    assert np.abs(got.astype(np.float64) - want.astype(np.float64)).max() <= (1e-12 if dtype == torch.float64 else 1e-6)
    assert (want > 0).all()


def test_nan_actor_raises_by_the_end_of_a_fused_iteration():
    pr = _problem(3, (64, 64, 64), torch.float32, update_backend="cuda", n_updates_per_iteration=2)
    with torch.no_grad():
        pr.models[1].actor.seq[0].weight[0, 0] = float("nan")
    tr = DSGDPPO(pr, DEV, {"alpha0": 1e-3, "mu": 0.0, "max_rl_timesteps": 10 ** 9, "writeout": False,
                           "consensus_backend": "fused"})
    _load(pr, _batch(pr, 64))
    pr.update_advantage()
    tr._consensus(0)
    assert tr.inner._program.capturable
    with pytest.raises(NameError, match="actor returning something weird"):
        pr.check_update()


def test_runs_past_the_schedule_horizon_raise():
    tr, _, _ = _run("dsgd", "wheel3", torch.float32, "fused", iters=1)
    tr.inner.k = tr.inner._program.eng.horizon - 2
    with pytest.raises(RuntimeError, match="horizon"):
        tr.inner.run_rounds(5)


@pytest.mark.parametrize("mod", ["train_cadmm_multi", "train_dsgd_multi", "train_dsgt_multi"])
def test_end_to_end(mod, tmp_path):
    import importlib
    from nn_distributed_training_b200.rl.train_common import make_problem, parse_args
    main = importlib.import_module(f"nn_distributed_training_b200.rl.{mod}").main
    base = ["--num_envs", "16", "--device", "cuda", "--rollout", "cuda", "--update", "cuda", "--seed", "0",
            "--max_rl_timesteps", "6000", "--save_freq", "1"]
    files = {}
    for backend in ("torch", "cuda"):
        out = tmp_path / backend
        main(base + ["--consensus", backend, "--out_dir", str(out)])
        files[backend] = sorted(os.listdir(out))
    assert files["cuda"] == files["torch"] and len(files["cuda"]) >= 5
    pr0, _ = make_problem(parse_args(base))                       # the seeded initial networks
    actors = [f for f in files["cuda"] if f.startswith("ppo_actors_tag_")]
    last = max(actors, key=lambda f: int(f.rsplit("_", 1)[1].split(".")[0]))
    sd = torch.load(tmp_path / "cuda" / last, map_location=DEV)
    for i in range(pr0.N):
        after = torch.nn.utils.parameters_to_vector(sd[f"actor{i}"].values())
        before = torch.nn.utils.parameters_to_vector(pr0.models[i].actor.state_dict().values())
        assert torch.isfinite(after).all() and not torch.equal(after, before)
    rews = np.load(tmp_path / "cuda" / [f for f in files["cuda"] if f.startswith("avg_ep_rews")][0])
    assert len(rews) >= 2 and np.isfinite(rews).all()
