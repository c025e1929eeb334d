"""GT-HSGD on the PyTorch path (CPU, float64): the NumPy oracle round by round on six graph kinds with and without link
drops, the tracking invariant, DSGT at beta = 1 bit for bit, exactness on heterogeneous least squares, the variance
reduction on noisy least squares, the same-minibatch gradient pair of the autograd path, every configuration refusal,
the runners and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import hsgd_oracle as ho
from test_exact_diffusion import GRAPHS as ED_GRAPHS, LeastSquares, _mnist_problem, _synthetic
from test_sgp import _exp
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, DSGT, GTHSGD
from nn_distributed_training_b200.problems.base import ConsensusProblem
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
GRAPHS = {
    "cycle": nx.cycle_graph(8),
    "path": nx.path_graph(6),
    "star": nx.star_graph(6),
    "wheel": nx.wheel_graph(7),
    "random": ED_GRAPHS["random"][0],
    "complete": nx.complete_graph(6),
}
BETAS = [1.0, 0.5, 0.1, 0.01]
DROPS = {"link_drop_prob": 0.3, "seed": 5, "from_round": 2, "to_round": 12}


def _conf(**kw):
    return dict({"alg_name": "gt_hsgd", "alpha": 0.05, "beta": 0.1, "outer_iterations": 50}, **kw)


class LSProblem(ConsensusProblem):
    """Heterogeneous least squares as a ConsensusProblem: node i holds ``m`` rows ``(a, b)`` of its own linear model plus
    noise, and its loss on a minibatch is the mean squared residual of ``Linear(n, 1, bias=False)``.  With
    ``batch == m`` every draw is the whole shard (full gradients in a permuted order)."""

    squeeze_output = True

    def __init__(self, graph, n=5, m=40, batch=40, noise=0.1, seed=0, faults=None):
        rng = np.random.default_rng(seed)
        N = graph.number_of_nodes()
        self.A = rng.standard_normal((N, m, n))
        x_own = 3.0 * rng.standard_normal((N, n))
        self.b = np.einsum("imn,in->im", self.A, x_own) + noise * rng.standard_normal((N, m))
        sets = [torch.utils.data.TensorDataset(torch.as_tensor(self.A[i]), torch.as_tensor(self.b[i])) for i in range(N)]
        torch.manual_seed(seed)
        conf = {"problem_name": "ls", "train_batch_size": batch, "val_batch_size": m, "metrics": [],
                "metrics_config": {"evaluate_frequency": 10 ** 9}}
        if faults:
            conf["fault_injection"] = dict(faults)
        super().__init__(graph, torch.nn.Linear(n, 1, bias=False).double(), torch.nn.MSELoss(), sets, None, "cpu",
                         conf, backend="torch", seed=seed)

    def evaluate_metrics(self, at_end=False):
        pass

    def solution(self):
        H = sum(self.A[i].T @ self.A[i] for i in range(self.N))
        r = sum(self.A[i].T @ self.b[i] for i in range(self.N))
        return np.linalg.solve(H, r)

    def batch_grad(self, x, k):
        """``[N, n]`` gradients of every node at points ``x`` on its draw k (the problem's sampler), in float64."""
        out = np.zeros_like(x)
        for i in range(self.N):
            idx = self.schedules[i].indices(k, self.seed, i).numpy()
            A, b = self.A[i][idx], self.b[i][idx]
            out[i] = 2.0 * A.T @ (A @ x[i] - b) / len(idx)
        return out


def _np(t, n=5):
    return t[:, :n].double().numpy().copy()


def _plan_W(pr, rounds):
    return [ho.metropolis(g) for g in pr.plan_graphs(rounds, 0, 1)]


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("drops", [False, True], ids=["static", "link_drops"])
@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph, beta, drops):
    R = 14
    pr = LSProblem(GRAPHS[graph], batch=8, seed=1, faults=DROPS if drops else None)
    Ws = _plan_W(pr, R)
    if drops:
        assert any(not np.array_equal(W, Ws[0]) for W in Ws)
    opt = GTHSGD(pr, "cpu", _conf(beta=beta, outer_iterations=R))
    ref = ho.run(_np(pr.arena.theta), Ws, 0.05, beta, pr.batch_grad, R)
    for k, (theta, y, v, tp) in enumerate(ref):
        opt.run_rounds(1)
        for name, got, want in (("theta", opt.arena.theta, theta), ("y", opt.y, y), ("v", opt.v, v),
                                ("theta_prev", opt.theta_prev, tp)):
            np.testing.assert_allclose(_np(got), want, rtol=1e-11, atol=1e-11, err_msg=f"round {k} {name}")
    assert pr.calls.tolist() == [R] * pr.N


@pytest.mark.parametrize("graph", ["cycle", "wheel", "random"])
def test_tracker_sum_equals_estimator_sum_every_round(graph):
    pr = LSProblem(GRAPHS[graph], batch=8, seed=5, faults=DROPS)
    opt = GTHSGD(pr, "cpu", _conf(beta=0.2))
    for k in range(20):
        opt.run_rounds(1)
        ys, vs = opt.y.sum(0), opt.v.sum(0)
        assert (ys - vs).abs().max().item() <= 1e-13 * max(1.0, opt.v.abs().max().item()), f"round {k}"


@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_beta_one_is_dsgt_bit_for_bit(model):
    """beta = 1: v' = g + 0 (v - gp) = g, so every round is DSGT's with init_grads false, bit for bit."""
    R = 12
    dconf = {"alg_name": "dsgt", "alpha": 0.05, "init_grads": False, "outer_iterations": R}
    hconf = _conf(beta=1.0, outer_iterations=R)
    if model == "mnist":
        pa, pb = _mnist_problem(hconf), _mnist_problem(dconf)
    else:
        pa, pb = LSProblem(GRAPHS["random"], batch=8, seed=2), LSProblem(GRAPHS["random"], batch=8, seed=2)
    a, b = GTHSGD(pa, "cpu", hconf), DSGT(pb, "cpu", dconf)
    assert a.omb == 0.0
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"
        assert torch.equal(a.y, b.y) and torch.equal(a.v, b.g), f"round {k}"
    assert pa.forward_cnt == pb.forward_cnt and (pa.calls == pb.calls).all()


def test_gt_hsgd_reaches_the_global_least_squares_solution_where_dsgd_does_not():
    """Heterogeneous least squares, full-batch gradients, cycle, constant step: GT-HSGD converges to the minimiser of
    sum_i f_i (with full batches gp is the exact gradient at theta_prev, so v = g after round 0); DSGD stops a
    measurable distance away."""
    rounds, alpha = 2000, 0.02
    pr = LSProblem(nx.cycle_graph(8), seed=3)
    opt = GTHSGD(pr, "cpu", _conf(alpha=alpha, beta=0.3, outer_iterations=rounds))
    opt.run_rounds(rounds)
    err = np.abs(_np(opt.arena.theta) - pr.solution()).max()
    pd = LSProblem(nx.cycle_graph(8), seed=3)
    od = DSGD(pd, "cpu", {"alg_name": "dsgd", "alpha0": alpha, "mu": 0.0, "outer_iterations": rounds})
    od.run_rounds(rounds)
    err_dsgd = np.abs(_np(od.arena.theta) - pd.solution()).max()
    print(f"\nmax |theta - x*| GT-HSGD {err:.2e}, DSGD {err_dsgd:.2e}")
    assert err < 1e-9
    assert err_dsgd > 1e-3


def test_variance_reduction_beats_dsgt_on_noisy_least_squares():
    """Heterogeneous noisy least squares with seeded minibatches of 2 rows out of 200: at the same constant step the
    tracked estimator's noise shrinks with beta, so GT-HSGD at a small beta ends closer to the minimiser than DSGT
    (mean squared distance over the last 500 of 3000 rounds)."""
    rounds, last, alpha = 3000, 500, 0.01
    out = {}
    for name in ("dsgt", "gt_hsgd"):
        pr = LSProblem(nx.cycle_graph(8), m=200, batch=2, noise=2.0, seed=4)
        x_star = pr.solution()
        if name == "dsgt":
            opt = DSGT(pr, "cpu", {"alg_name": "dsgt", "alpha": alpha, "init_grads": False, "outer_iterations": rounds})
        else:
            opt = GTHSGD(pr, "cpu", _conf(alpha=alpha, beta=0.05, outer_iterations=rounds))
        msd = []
        for k in range(rounds):
            opt.run_rounds(1)
            if k >= rounds - last:
                msd.append(((_np(opt.arena.theta) - x_star) ** 2).sum(1).mean())
        out[name] = float(np.mean(msd))
    print(f"\nmean squared distance to x* over the last {last} rounds: DSGT {out['dsgt']:.4e}, "
          f"GT-HSGD (beta 0.05) {out['gt_hsgd']:.4e}")
    assert out["gt_hsgd"] < out["dsgt"]


# ----------------------------------------------------------------------------------- same-minibatch pair ----
@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_compute_grads_pair_equals_two_autograd_calls_on_the_same_indices(model):
    if model == "mnist":
        pr = _mnist_problem(_conf())
    else:
        pr = LSProblem(GRAPHS["wheel"], batch=8, seed=6)
    pr.count_draws_all(3)                    # a draw other than the first
    calls, fwd = pr.calls.copy(), pr.forward_cnt
    g = torch.Generator().manual_seed(0)
    theta_prev = pr.arena.theta + 0.01 * torch.randn(pr.arena.theta.shape, generator=g, dtype=pr.dtype)
    theta_prev[:, pr.n:] = 0
    grad_prev = pr.arena.zeros()
    pr.compute_grads_pair(theta_prev, grad_prev)
    assert (pr.calls == calls + 1).all() and pr.forward_cnt == fwd + pr.train_batch_size
    for point, got in ((pr.arena.theta, pr.arena.grad), (theta_prev, grad_prev)):
        for l in range(pr.N):
            m = copy.deepcopy(pr.models[l])
            for p, v in zip(m.parameters(), pr.layout.views(point[l])):
                p.data = v.clone()
            idx = pr.schedules[l].indices(int(calls[l]), pr.seed, l)
            sh = pr.shards.shard(l)
            loss = pr._loss(m, sh.inputs(idx, pr.dtype), sh.targets(idx))
            want = torch.cat([t.reshape(-1) for t in torch.autograd.grad(loss, list(m.parameters()))])
            assert torch.equal(pr.arena.compact(got[l:l + 1])[0], want), l


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "gt_hsgd", "alpha": 0.01, "beta": 0.1, "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["gt_hsgd"] is GTHSGD
    c = validate_optimizer(dict(BASE))
    assert c["update_graph"] is True and c["profile"] is False
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, beta=1.0, update_graph=False, profile=True))


@pytest.mark.parametrize("key", ["alpha", "beta", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})


@pytest.mark.parametrize("alpha", [0.0, -0.1, float("inf"), float("nan"), "0.1", True])
def test_alpha_must_be_finite_and_positive(alpha):
    with pytest.raises(ConfigError, match="alpha"):
        validate_optimizer(dict(BASE, alpha=alpha))
    if not isinstance(alpha, (str, bool)):
        with pytest.raises(ValueError, match="alpha"):
            GTHSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(alpha=alpha))


@pytest.mark.parametrize("beta", [0.0, -0.5, 1.5, float("inf"), float("nan"), "0.5", True])
def test_beta_must_be_finite_and_in_zero_one(beta):
    with pytest.raises(ConfigError, match="beta"):
        validate_optimizer(dict(BASE, beta=beta))
    with pytest.raises(ValueError, match="beta"):
        GTHSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(beta=beta))


@pytest.mark.parametrize("key", ["mu", "init_grads", "gamma", "gossip_steps"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"gt_hsgd takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        GTHSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        GTHSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'gt_hsgd'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        GTHSGD(LSProblem(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())


def test_reference_api_problem_is_refused():
    """A problem behind the reference API draws its minibatch inside local_batch_loss and cannot replay it."""
    with pytest.raises(ValueError, match="same minibatch"):
        GTHSGD(LeastSquares([GRAPHS["cycle"]]), "cpu", _conf())


def test_changing_graphs_and_link_drops_are_accepted():
    """The tracking invariant holds for any doubly stochastic W: a graph that changes every round runs."""
    pr = LSProblem(GRAPHS["cycle"], faults=dict(DROPS, from_round=0, to_round=6))
    assert len({tuple(sorted(g.edges())) for g in pr.plan_graphs(6, 0, 1)}) > 1
    GTHSGD(pr, "cpu", _conf(outer_iterations=6)).run_rounds(6)
    assert np.isfinite(pr.arena.theta.numpy()).all()


# ------------------------------------------------------------------------------------------------ runners ----
def test_gt_hsgd_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_hsgd.yaml"), "mnist")
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [(o["alg_name"], o.get("beta")) for o in ocs] == [("dsgt", None), ("gt_hsgd", 0.3), ("gt_hsgd", 0.1)]
    assert all(o["alpha"] == 0.005 for o in ocs)
    paper = load_experiment(os.path.join(EXP, "dist_mnist_detag.yaml"), "mnist")
    assert dict(conf["experiment"], name=None) == dict(paper["experiment"], name=None)


def test_mnist_runner_on_the_hsgd_yaml(tmp_path, monkeypatch):
    """The three problems of the YAML at a tiny size; GT-HSGD draws one batch per round."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_hsgd.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True, use_cuda=False)
    conf["experiment"]["graph"]["num_nodes"] = 4
    for pc in conf["problem_configs"].values():
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"]["outer_iterations"] = 3
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_hsgd"))
    assert len(out) == 1
    res = {}
    for name in ("dsgt", "gt_hsgd_b0.3", "gt_hsgd_b0.1"):
        res[name] = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert all(torch.isfinite(v).all() for v in res[name]["validation_loss"])
    fp = {k: [int(torch.as_tensor(v).sum()) for v in r["forward_pass_count"]] for k, r in res.items()}
    assert fp["gt_hsgd_b0.3"] == fp["gt_hsgd_b0.1"] == fp["dsgt"]


def test_density_runner_runs_gt_hsgd(tmp_path):
    from test_runners import _small_density_conf, _write, synthetic_dir  # noqa: F401
    from nn_distributed_training_b200.experiments import dist_dense_ex
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path / "floor")
    os.makedirs(d)
    write_dataset(d, n_paths=4, seed=0)
    conf = _small_density_conf("dist_dense_v2.yaml", d, tmp_path)
    conf["experiment"]["graph"].update(num_nodes=3, p=0.9)
    conf["experiment"]["individual_training"]["train_solo"] = False
    pc = conf["problem_configs"]["problem1"]
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="gt_hsgd")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "gt_hsgd", "alpha": 0.01, "beta": 0.2, "outer_iterations": 4}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "gt_hsgd_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha=0.02, beta=0.3, outer_iterations=6)
    full = _mnist_problem(conf)
    of = GTHSGD(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = GTHSGD(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = GTHSGD(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3
    for name in ("y", "v", "theta_prev"):
        assert torch.equal(getattr(o2, name), getattr(o1, name)), name
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in ("y", "v", "theta_prev"):
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt
