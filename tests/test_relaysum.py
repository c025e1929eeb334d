"""RelaySum on the PyTorch path (CPU): the float64 oracle of ``tests/relaysum_oracle.py`` round by round on paths, stars,
binary trees and a random tree, the reach table against the relayed-count recursion, the delayed-sum closed form, round 0
as the identity, the 2-node equivalence with DSGD, exactness on heterogeneous least squares, the refusals,
configuration, the runners and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import relaysum_oracle as ro
from test_exact_diffusion import LeastSquares, _synthetic
from test_sgp import _exp
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, RelaySum
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer
from nn_distributed_training_b200.utils.graph_generation import Topology, generate_from_conf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


def _gen(kind, N):
    return generate_from_conf({"type": kind, "num_nodes": N})[1]


def _prufer_tree():
    rng = np.random.default_rng(11)
    return nx.from_prufer_sequence([int(x) for x in rng.integers(0, 9, size=7)])


TREES = {
    "path2": _gen("path", 2), "path6": _gen("path", 6), "path10": _gen("path", 10),
    "star5": _gen("star", 5), "star10": _gen("star", 10),
    "binary_tree7": _gen("binary_tree", 7), "binary_tree10": _gen("binary_tree", 10),
    "prufer9": _prufer_tree(),
}


def _conf(**kw):
    return dict({"alg_name": "relaysum", "alpha0": 0.05, "mu": 0.0, "outer_iterations": 40}, **kw)


def _theta(opt, n=5):
    return opt.arena.theta[:, :n].double().numpy().copy()


# ------------------------------------------------------------------------------------------------ graphs ----
def test_binary_tree_kind_and_its_children():
    g = _gen("binary_tree", 10)
    assert nx.is_tree(g) and g.number_of_nodes() == 10
    for i in range(10):
        kids = {c for c in (2 * i + 1, 2 * i + 2) if c < 10}
        assert kids <= set(g.neighbors(i))
    assert Topology(g).is_tree()
    assert not Topology(nx.cycle_graph(5)).is_tree()
    assert not Topology(nx.Graph([(0, 1), (2, 3), (3, 4)])).is_tree()


@pytest.mark.parametrize("name", sorted(TREES))
def test_reverse_slots(name):
    t = Topology(TREES[name])
    rs = t.reverse_slots()
    for i, nb in enumerate(t.neighbors_noself):
        for e, j in enumerate(nb):
            assert t.neighbors_noself[j][rs[i][e]] == i


@pytest.mark.parametrize("name", sorted(TREES))
def test_reach_table_equals_the_relayed_count_recursion(name):
    """``R_i^k - 1`` from breadth-first search equals ``sum_j c_{j->i}`` of the recursion
    ``c_{i->j} = 1 + sum_{l != j} c_{l->i}``, exactly in integers, for every round (past the diameter too)."""
    t = Topology(TREES[name])
    R = t.reach_table()
    assert R.shape[1] == 1 + max(nx.eccentricity(TREES[name]).values())
    counts = ro.relayed_counts(t.neighbors_noself)
    for k in range(counts.shape[1]):
        assert np.array_equal(R[:, min(k, R.shape[1] - 1)] - 1, counts[:, k]), f"round {k}"
    assert (R[:, -1] == t.N).all()


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("mu", [0.0, 0.5])
@pytest.mark.parametrize("name", sorted(TREES))
def test_torch_path_matches_float64_oracle_round_by_round(name, mu):
    g = TREES[name]
    pr = LeastSquares([g], seed=1)
    opt = RelaySum(pr, "cpu", _conf(mu=mu))
    nbrs = Topology(g).neighbors_noself
    dist = ro.hop_distances(nbrs)
    h, msg = _theta(opt), {}
    alphas = opt.alpha_table(14)
    for k in range(14):
        opt.run_rounds(1)
        h, msg, _ = ro.round_(h, msg, k, nbrs, dist, pr.grad, alphas[k])
        np.testing.assert_allclose(_theta(opt), h, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        for (i, j), m in msg.items():
            e = nbrs[i].index(j)
            np.testing.assert_allclose(opt.msg[i, e, :5].numpy(), m, rtol=1e-12, atol=1e-12,
                                       err_msg=f"round {k}: m_{i}->{j}")
        for i in range(pr.N):
            assert not opt.msg[i, len(nbrs[i]):].any()


@pytest.mark.parametrize("name", ["path10", "star10", "binary_tree10", "prufer9"])
def test_mix_is_the_delayed_sum_of_the_recorded_half_steps(name):
    """``x_i^(k) = h_i^(k-1) + (1/n) sum_{l != i, d(i,l) <= k} (h_l^(k - d(i,l)) - h_i^(k-1))`` against a recorded
    history of h (``h^(k)`` after round k, ``h^(-1)`` the initial parameters)."""
    g = TREES[name]
    pr = LeastSquares([g], seed=2)
    nbrs = Topology(g).neighbors_noself
    dist = ro.hop_distances(nbrs)
    N = pr.N
    hist = {-1: _theta(RelaySum(pr, "cpu", _conf()))}
    msg = {}
    for k in range(12):
        h_new, msg, x = ro.round_(hist[k - 1], msg, k, nbrs, dist, pr.grad, 0.05)
        want = np.zeros_like(x)
        for i in range(N):
            want[i] = hist[k - 1][i] + sum((hist[k - dist[i, l]][l] - hist[k - 1][i]
                                            for l in range(N) if l != i and dist[i, l] <= k), np.zeros(x.shape[1])) / N
        np.testing.assert_allclose(x, want, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        hist[k] = h_new


@pytest.mark.parametrize("name", ["path6", "star10", "binary_tree7"])
def test_round_zero_is_the_identity(name):
    """With every message zero and R_i^0 - 1 = 0 the mix leaves theta bitwise as it was: round 0 is a plain SGD step."""
    pr = LeastSquares([TREES[name]], seed=3)
    opt = RelaySum(pr, "cpu", _conf())
    seen = {}
    orig = pr.batched_grads

    def spy(views):
        seen["x"] = opt.arena.theta.clone()
        return orig(views)
    pr.batched_grads = spy
    before = opt.arena.theta.clone()
    opt.run_rounds(1)
    assert torch.equal(seen["x"], before)


def test_two_nodes_equal_dsgd_from_round_one():
    """On ``path`` 2 the Metropolis weights are 1/2 and from round 1 on each node averages its own h with the other's, as
    DSGD does; round 0 differs (the identity, not the average), so both start from the row after round 0."""
    g = nx.path_graph(2)
    pr_r, pr_d = LeastSquares([g], seed=4), LeastSquares([g], seed=4)
    o_r, o_d = RelaySum(pr_r, "cpu", _conf()), DSGD(pr_d, "cpu", _conf(alg_name="dsgd"))
    o_r.run_rounds(1)
    o_d.k = o_r.k
    o_d.alph = o_r.alph
    o_d.arena.theta.copy_(o_r.arena.theta)
    for k in range(1, 30):
        o_r.run_rounds(1)
        o_d.run_rounds(1)
        np.testing.assert_allclose(_theta(o_r), _theta(o_d), rtol=1e-12, atol=1e-12, err_msg=f"round {k}")


def _distance(opt_cls, g, conf, rounds, seed=5):
    """The worst node's relative distance to the minimiser, at the rows the last round's gradients are taken at (the
    mixed x: between rounds a node holds x - alpha g_i)."""
    pr = LeastSquares([g], seed=seed)
    opt = opt_cls(pr, "cpu", dict(conf, outer_iterations=rounds))
    opt.run_rounds(rounds - 1)
    seen, orig = {}, pr.batched_grads

    def spy(views):
        seen["x"] = _theta(opt)
        return orig(views)
    pr.batched_grads = spy
    opt.run_rounds(1)
    xs = pr.solution()
    return max(np.linalg.norm(seen["x"][i] - xs) for i in range(pr.N)) / np.linalg.norm(xs)


@pytest.mark.parametrize("name", ["path10", "star10", "binary_tree10"])
def test_relaysum_reaches_the_minimiser_where_dsgd_does_not(name):
    """Heterogeneous least squares with full gradients and a constant step (alpha 0.05, 3000 rounds): every RelaySum node
    ends at the minimiser of sum_i f_i up to round-off, DSGD's nodes stay away from it (DESIGN §2.10 records both)."""
    g = TREES[name]
    relay = _distance(RelaySum, g, _conf(), 3000)
    dsgd = _distance(DSGD, g, _conf(alg_name="dsgd"), 3000)
    print(f"\n{name}: worst node's relative distance to the minimiser: relaysum {relay:.2e}, dsgd {dsgd:.2e}")
    assert relay < 1e-9
    assert dsgd > 1e-2


# ---------------------------------------------------------------------------------------------- refusals ----
def test_a_graph_that_is_not_a_tree_is_refused():
    for g in (nx.cycle_graph(5), nx.Graph([(0, 1), (2, 3), (3, 4)]), nx.complete_graph(4)):
        with pytest.raises(ValueError, match="relaysum needs a tree"):
            RelaySum(LeastSquares([g]), "cpu", _conf())
    RelaySum(LeastSquares([nx.complete_graph(2)]), "cpu", _conf())       # two nodes: a tree


def test_a_directed_graph_is_refused():
    with pytest.raises(ValueError, match="undirected"):
        RelaySum(LeastSquares([nx.path_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())
    conf = _exp("directed_cycle")
    conf["problem_configs"]["problem1"]["optimizer_config"] = _conf(outer_iterations=3)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'relaysum'"):
        validate_experiment(conf, "mnist")


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order: relaysum runs the synchronous 'jacobi' order only"):
        validate_optimizer(_conf(mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        RelaySum(LeastSquares([nx.path_graph(4)]), "cpu", _conf(mixing_order="reference"))


def test_link_drop_fault_injection_is_refused():
    pr = _mnist_problem(_conf(), graph=nx.path_graph(4))
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 6}
    pr._init_faults()
    with pytest.raises(ValueError, match="link-drop fault_injection"):
        RelaySum(pr, "cpu", _conf())


def test_a_graph_that_changes_during_the_run_is_refused():
    pr = LeastSquares([nx.path_graph(6), nx.star_graph(5)])
    opt = RelaySum(pr, "cpu", _conf())
    with pytest.raises(ValueError, match="fixed tree"):
        opt.run_rounds(2)


def test_a_multi_topology_plan_is_refused():
    """The moving online-density plan: a graph sequence of more than one topology is refused before the first round."""
    pr = _mnist_problem(_conf(), graph=nx.path_graph(4))
    pr.plan_graphs = lambda oits, k0, dpr, init_draws=0, refresh=True: [nx.path_graph(4), nx.star_graph(3)] * oits
    opt = RelaySum(pr, "cpu", _conf())
    with pytest.raises(ValueError, match="relaysum needs a fixed graph"):
        opt.train()


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "relaysum", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 3}


def test_registered_and_config_keys():
    assert ALGORITHMS["relaysum"] is RelaySum
    c = validate_optimizer(dict(BASE))
    assert c["profile"] is False
    for key in ("alpha0", "mu", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in BASE.items() if k != key})
    for key in ("update_graph", "consensus_backend", "checkpoint_every", "resume"):
        validate_optimizer(dict(BASE, **{key: True}))
    for key in ("beta", "momentum", "gamma", "alpha"):
        with pytest.raises(ConfigError, match=f"relaysum takes no key '{key}'"):
            validate_optimizer(dict(BASE, **{key: 0.5}))
    for a0 in (0.0, -1.0, "0.1", True):
        with pytest.raises(ConfigError, match="alpha0 must be > 0"):
            validate_optimizer(dict(BASE, alpha0=a0))
    with pytest.raises(ConfigError, match="mu must be >= 0"):
        validate_optimizer(dict(BASE, mu=-0.1))


def test_binary_tree_in_config_validation():
    conf = _exp("binary_tree")
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    validate_experiment(conf, "mnist")
    conf = load_experiment(os.path.join(EXP, "dist_mnist_relaysum.yaml"), "mnist")
    assert conf["experiment"]["graph"]["type"] == "binary_tree"
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [o["alg_name"] for o in ocs] == ["dsgd", "dsgt", "relaysum"]
    assert {o.get("alpha0", o.get("alpha")) for o in ocs} == {0.005}
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    for key in ("model", "data_split_type"):
        assert conf["experiment"][key] == paper["experiment"][key]


def test_checkpoint_carries_the_messages():
    opt = RelaySum(LeastSquares([TREES["binary_tree7"]]), "cpu", _conf())
    assert opt.STATE == ("msg",) and opt.msg.shape == (7, 3, opt.arena.n_pad) and not opt.msg.any()
    assert set(opt.state_dict()) == {"k", "theta", "msg", "alph"}


# ------------------------------------------------------------------------------------------------ runners ----
def test_mnist_runner_on_the_relaysum_yaml(tmp_path, monkeypatch):
    """The three problems of the new YAML on the binary tree, at a tiny size, through the MNIST runner."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_relaysum.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True, use_cuda=False)
    conf["experiment"]["graph"]["num_nodes"] = 5
    for pc in conf["problem_configs"].values():
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"]["outer_iterations"] = 3
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_relaysum"))
    assert len(out) == 1
    for name in ("dsgd", "dsgt", "relaysum"):
        res = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert len(res["validation_loss"]) == 2
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])


def test_density_runner_runs_relaysum_on_a_tree(tmp_path):
    from test_runners import _small_density_conf, _write, synthetic_dir  # noqa: F401
    from nn_distributed_training_b200.experiments import dist_dense_ex
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path / "floor")
    os.makedirs(d)
    write_dataset(d, n_paths=4, seed=0)
    conf = _small_density_conf("dist_dense_v2.yaml", d, tmp_path)
    conf["experiment"]["graph"] = {"type": "binary_tree", "num_nodes": 3}
    conf["experiment"]["individual_training"]["train_solo"] = False
    pc = conf["problem_configs"]["problem1"]
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="relaysum")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = dict(BASE, outer_iterations=4)
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "relaysum_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def _mnist_problem(conf, N=4, M=100, graph=None):
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
    return DistMNISTProblem(graph if graph is not None else nx.path_graph(N), MNISTConvNet(3, 5, 64),
                            torch.nn.NLLLoss(), shards, val, "cpu", pconf, backend="torch", seed=7)


def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, outer_iterations=6)
    g = nx.star_graph(3)
    full = _mnist_problem(conf, graph=g)
    of = RelaySum(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf, graph=g)
    o1 = RelaySum(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf, graph=g)
    o2 = RelaySum(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and o2.alph == o1.alph
    assert torch.equal(o2.msg, o1.msg) and o2.msg.any()
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.msg, of.msg)
    assert second.forward_cnt == full.forward_cnt
