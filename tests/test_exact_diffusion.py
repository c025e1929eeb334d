"""Exact Diffusion on the PyTorch path (CPU): a float64 oracle written from the algorithm's four steps, exactness on
local least-squares problems with different minimisers, configuration, the MNIST runner and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, ExactDiffusion
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


# ------------------------------------------------------------------------------------------------ oracle ----
def metropolis(g):
    """W_ij = 1 / (1 + max(d_i, d_j)) on edges, W_ii = 1 - sum_j W_ij."""
    N = g.number_of_nodes()
    d = np.array([g.degree(i) for i in range(N)], dtype=np.float64)
    W = np.zeros((N, N))
    for i, j in g.edges():
        if i != j:
            W[i, j] = W[j, i] = 1.0 / (1.0 + max(d[i], d[j]))
    W[np.diag_indices(N)] = 1.0 - W.sum(1)
    return W


def oracle_round(theta, psi, k, W, grad_fn, alpha):
    """Round k of every node: mix with A = (I + W) / 2, psi = theta at k = 0, adapt, correct."""
    N = theta.shape[0]
    mixed = np.zeros_like(theta)
    for i in range(N):
        mixed[i] = 0.5 * (1.0 + W[i, i]) * theta[i]
        for j in range(N):
            if j != i and W[i, j] != 0.0:
                mixed[i] += 0.5 * W[i, j] * theta[j]
    if k == 0:
        psi = mixed.copy()
    new_psi = np.stack([mixed[i] - alpha * grad_fn(i, mixed[i]) for i in range(N)])
    return new_psi + (mixed - psi), new_psi


# ---------------------------------------------------------------------------------------- least squares ----
class LeastSquares:
    """Node i minimises 0.5 / m |A_i x - b_i|^2 with its own minimiser; exact gradients for every node in one call.
    ``graphs`` of more than one entry: ``update_graph`` steps through them (a graph that changes every round)."""

    capturable_grads = False

    def __init__(self, graphs, n=5, m=20, seed=0, dtype=torch.float64):
        rng = np.random.default_rng(seed)
        self.graphs = graphs
        self.idx = 0
        self.graph = graphs[0]
        self.N = self.graph.number_of_nodes()
        self.A = rng.standard_normal((self.N, m, n))
        x_own = 3.0 * rng.standard_normal((self.N, n))
        self.b = np.einsum("imn,in->im", self.A, x_own) + 0.1 * rng.standard_normal((self.N, m))
        self.m = m
        torch.manual_seed(seed)
        self.models = [torch.nn.Linear(n, 1, bias=False).to(dtype) for _ in range(self.N)]
        self.conf = {"metrics_config": {"evaluate_frequency": 10 ** 9}}
        self._A = torch.as_tensor(self.A, dtype=dtype)
        self._b = torch.as_tensor(self.b, dtype=dtype)

    def grad(self, i, x):
        return self.A[i].T @ (self.A[i] @ x - self.b[i]) / self.m

    def solution(self):
        H = sum(self.A[i].T @ self.A[i] for i in range(self.N))
        r = sum(self.A[i].T @ self.b[i] for i in range(self.N))
        return np.linalg.solve(H, r)

    def update_graph(self):
        self.idx += 1
        self.graph = self.graphs[self.idx % len(self.graphs)]

    def batched_grads(self, views):
        x = torch.stack([m.weight.detach().reshape(-1) for m in self.models])
        r = torch.einsum("imn,in->im", self._A, x) - self._b
        g = torch.einsum("imn,im->in", self._A, r) / self.m
        for i in range(self.N):
            views[i][0].copy_(g[i].reshape(1, -1))
        return 0.5 * (r * r).mean(1, keepdim=True)

    def evaluate_metrics(self, at_end=False):
        pass


def _isolated():
    g = nx.Graph([(0, 1), (1, 2), (2, 3), (3, 0), (0, 2), (4, 5)])
    g.add_node(6)
    return nx.convert_node_labels_to_integers(g)


def _random():
    for seed in range(1000):
        g = nx.gnp_random_graph(7, 0.45, seed=seed)
        if nx.is_connected(g):
            return g
    raise AssertionError("no connected random graph")


GRAPHS = {
    "cycle": [nx.cycle_graph(6)],
    "wheel": [nx.wheel_graph(7)],
    "complete": [nx.complete_graph(6)],
    "random": [_random()],
    "isolated": [_isolated()],
    "switching": [nx.cycle_graph(6), nx.star_graph(5), nx.complete_graph(6), nx.path_graph(6), nx.empty_graph(6)],
}


def _conf(**kw):
    return dict({"alg_name": "exact_diffusion", "alpha0": 0.05, "mu": 0.0, "outer_iterations": 50}, **kw)


def _theta(opt):
    return opt.arena.theta[:, :opt.pr.layout.n].double().numpy().copy()


@pytest.mark.parametrize("mu", [0.0, 0.7])
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph, mu):
    pr = LeastSquares(GRAPHS[graph], seed=1)
    opt = ExactDiffusion(pr, "cpu", _conf(mu=mu))
    theta, psi = _theta(opt), None
    alpha = 0.05
    for k in range(8):
        opt.run_rounds(1)
        alpha = alpha * (1.0 - mu * alpha)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        theta, psi = oracle_round(theta, psi, k, W, pr.grad, alpha)
        np.testing.assert_allclose(_theta(opt), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        np.testing.assert_allclose(opt.psi[:, :5].numpy(), psi, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
    assert opt.alph == pytest.approx(alpha, rel=1e-15)


def test_isolated_node_takes_plain_sgd_steps():
    """A node without neighbours: theta == psi after every round, so each round is exactly one SGD step."""
    pr = LeastSquares(GRAPHS["isolated"], seed=2)
    opt = ExactDiffusion(pr, "cpu", _conf())
    x = _theta(opt)[6]
    for _ in range(5):
        opt.run_rounds(1)
        x = x - 0.05 * pr.grad(6, x)
        assert np.array_equal(_theta(opt)[6], opt.psi[6, :5].numpy())
    np.testing.assert_allclose(_theta(opt)[6], x, rtol=1e-13, atol=1e-14)


def test_exact_diffusion_reaches_the_global_least_squares_solution():
    """Static 8-node cycle, 5 unknowns, 20 rows per node, exact gradients, constant alpha = 0.05: Exact Diffusion
    converges to the minimiser of the summed losses to round-off; DSGD at the same step stays biased."""
    g = [nx.cycle_graph(8)]
    rounds = 5000
    pr = LeastSquares(g, seed=3)
    x_star = pr.solution()
    ed = ExactDiffusion(pr, "cpu", _conf(outer_iterations=rounds))
    ed.run_rounds(rounds)
    err_ed = np.abs(_theta(ed) - x_star).max()
    pr2 = LeastSquares(g, seed=3)
    dsgd = DSGD(pr2, "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.0, "outer_iterations": rounds})
    dsgd.run_rounds(rounds)
    err_dsgd = np.abs(_theta(dsgd) - x_star).max()
    print(f"\n|theta - x*|_max after {rounds} rounds: exact diffusion {err_ed:.3e}, dsgd {err_dsgd:.3e}")
    assert err_ed < 1e-9 * max(1.0, np.abs(x_star).max())
    assert err_dsgd > 100 * err_ed and err_dsgd > 1e-3


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["exact_diffusion"] is ExactDiffusion
    c = validate_optimizer({"alg_name": "exact_diffusion", "alpha0": 0.01, "outer_iterations": 3})
    assert c["mu"] == 0.0 and c["profile"] is False
    with pytest.raises(ConfigError, match="alpha0"):
        validate_optimizer({"alg_name": "exact_diffusion", "outer_iterations": 3})
    with pytest.raises(ConfigError, match="outer_iterations"):
        validate_optimizer({"alg_name": "exact_diffusion", "alpha0": 0.01})
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer({"alg_name": "exact_diffusion", "alpha0": 0.01, "outer_iterations": 3,
                            "mixing_order": "reference"})
    for key in ("update_graph", "consensus_backend", "checkpoint_every", "resume"):
        validate_optimizer({"alg_name": "exact_diffusion", "alpha0": 0.01, "outer_iterations": 3, key: True})
    with pytest.raises(ValueError, match="jacobi"):
        ExactDiffusion(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_hetero_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_hetero_ed.yaml"), "mnist")
    algs = [p["optimizer_config"]["alg_name"] for p in conf["problem_configs"].values()]
    assert algs == ["exact_diffusion", "dsgt", "dsgd"]
    assert conf["experiment"]["data_split_type"] == "hetero"
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    for key in ("graph", "model", "data_split_type"):
        assert conf["experiment"][key] == paper["experiment"][key]


# ------------------------------------------------------------------------------------------------ runner ----
def _synthetic(monkeypatch):
    import nn_distributed_training_b200.data.mnist as M
    from nn_distributed_training_b200.experiments import dist_mnist_ex
    monkeypatch.setattr(M, "load_mnist", lambda d, train, **k: (M.synthetic_mnist(512 if train else 128, seed=int(train)), "synthetic"))
    monkeypatch.setattr(dist_mnist_ex, "load_mnist", M.load_mnist)
    return dist_mnist_ex


def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="exact_diffusion")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "exact_diffusion", "alpha0": 0.01, "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    files = set(os.listdir(outs[0]))
    assert {"graph.gpickle", "exact_diffusion_results.pt"} <= files
    res = torch.load(os.path.join(outs[0], "exact_diffusion_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"}
    assert len(res["validation_loss"]) == 3          # rounds 0, 2 and 4 (the last)
    assert res["validation_loss"][0].shape == (2,)
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def _mnist_problem(conf, N=4, M=100):
    from nn_distributed_training_b200.data.mnist import synthetic_mnist
    from nn_distributed_training_b200.models import MNISTConvNet
    from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem
    torch.manual_seed(0)
    data = synthetic_mnist(M * N, seed=3)
    val = synthetic_mnist(64, seed=4)
    shards = [data.select(torch.arange(i * M, (i + 1) * M)) for i in range(N)]
    pconf = {"problem_name": "t", "train_batch_size": 32, "val_batch_size": 64,
             "metrics": ["forward_pass_count", "validation_loss"], "metrics_config": {"evaluate_frequency": 1000},
             "optimizer_config": conf}
    return DistMNISTProblem(nx.wheel_graph(N), MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, val, "cpu",
                            pconf, backend="torch", seed=7)


def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, outer_iterations=6)
    full = _mnist_problem(conf)
    of = ExactDiffusion(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = ExactDiffusion(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = ExactDiffusion(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.psi, o1.psi)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.psi, of.psi)
    assert o2.alph == of.alph
    assert second.forward_cnt == full.forward_cnt
