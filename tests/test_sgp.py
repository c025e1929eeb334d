"""SGP (push-sum SGD) on the PyTorch path (CPU): the directed graph generators and push-sum weights, a float64 oracle
round by round on directed, irregular undirected and changing graphs, the push-sum invariants and why the de-biasing
matters, DSGD equivalence on the cycle, convergence on a heterogeneous problem, configuration, the MNIST runner and
checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import sgp_oracle as so
from test_exact_diffusion import LeastSquares, metropolis
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, SGP
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer
from nn_distributed_training_b200.utils.graph_generation import Topology, adjacency, generate_from_conf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


def _gen(kind, N, **kw):
    return generate_from_conf(dict({"type": kind, "num_nodes": N}, **kw))[1]


def _conf(**kw):
    return dict({"alg_name": "sgp", "alpha0": 0.05, "mu": 0.0, "outer_iterations": 50}, **kw)


def _switching():
    """A different digraph every round, none of them strongly connected on its own."""
    gs = []
    for k in range(4):
        g = nx.DiGraph()
        g.add_nodes_from(range(6))
        g.add_edges_from((i, (i + k + 1) % 6) for i in range(0, 6, 2))
        g.add_edge(5, k + 1)
        gs.append(g)
    return gs


GRAPHS = {
    "directed_cycle": [_gen("directed_cycle", 6)],
    "exponential": [_gen("exponential", 7)],
    "random_directed": [_gen("random_directed", 7, p=0.3, seed=2, gen_attempts=200)],
    "wheel": [nx.wheel_graph(7)],
    "star": [nx.star_graph(5)],
    "switching": _switching(),
}


# ------------------------------------------------------------------------------------------------ graphs ----
def test_directed_generators_degrees_and_strong_connectivity():
    g = _gen("directed_cycle", 6)
    assert g.is_directed() and sorted(g.edges()) == [(i, (i + 1) % 6) for i in range(6)]
    for N, m in ((10, 4), (8, 3), (5, 3), (2, 1)):
        g = _gen("exponential", N)
        assert all(g.out_degree(i) == m and g.in_degree(i) == m for i in range(N)), N
        assert all(g.has_edge(i, (i + 4) % N) for i in range(N)) == (N > 4)
    for seed in range(5):
        g = _gen("random_directed", 9, p=0.25, seed=seed, gen_attempts=500)
        assert nx.is_strongly_connected(g)
        assert Topology(g).is_connected()
    with pytest.raises(NameError, match="strongly connected"):
        _gen("random_directed", 9, p=0.0, seed=0, gen_attempts=3)
    # one-way path: weakly but not strongly connected
    assert not Topology(nx.DiGraph([(0, 1), (1, 2)])).is_connected()


@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_topology_tables_and_push_weights(graph):
    for g in GRAPHS[graph]:
        t = Topology(g)
        A = so.column_stochastic(g)
        np.testing.assert_array_equal(t.push_weights, A)
        np.testing.assert_allclose(t.push_weights.sum(0), 1.0, rtol=0, atol=1e-15)
        ins, _ = so.pull_lists(g)
        assert [sorted(n) for n in t.neighbors_noself] == ins
        if g.is_directed():
            assert t.W is None and t.directed
            assert [sorted(r) for r in t.readers] == [sorted(g.successors(i)) for i in range(t.N)]
            assert list(t.deg) == [g.in_degree(i) for i in range(t.N)]
        else:
            np.testing.assert_array_equal(t.W, metropolis(g))
            assert t.readers == t.neighbors_noself


def test_undirected_adjacency_unchanged_and_directed_keeps_direction():
    g = nx.path_graph(3)
    a = adjacency(g)
    assert a[0, 1] and a[1, 0] and not a[0, 2]
    d = adjacency(nx.DiGraph([(0, 1), (1, 2)]))
    assert d[0, 1] and not d[1, 0]
    # the same edge set directed both ways is not the undirected topology
    both = nx.DiGraph([(0, 1), (1, 0), (1, 2), (2, 1)])
    assert Topology(both).key != Topology(g).key


# ------------------------------------------------------------------------------------------------ oracle ----
def _x(opt):
    return opt.x.double().numpy()[:, :5].copy()


@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph):
    gs = GRAPHS[graph]
    pr = LeastSquares(gs, seed=1)
    opt = SGP(pr, "cpu", _conf(mu=0.5))
    x = _x(opt)
    w = np.ones(pr.N)
    alpha = 0.05
    for k in range(10):
        g = gs[(pr.idx + 1) % len(gs)]          # the round refreshes the graph first
        opt.run_rounds(1)
        alpha = alpha * (1.0 - 0.5 * alpha)
        x, w, th = so.sgp_round(x, w, g, pr.grad, alpha)
        np.testing.assert_allclose(_x(opt), x, rtol=1e-12, atol=1e-13, err_msg=f"round {k} x")
        np.testing.assert_allclose(opt.w.numpy(), w, rtol=1e-14, atol=0, err_msg=f"round {k} w")
        np.testing.assert_allclose(opt.arena.theta.numpy()[:, :5], th, rtol=1e-12, atol=1e-13, err_msg=f"round {k} theta")
    if graph in ("wheel", "star", "random_directed"):
        assert np.abs(w - 1.0).max() > 1e-2          # not doubly stochastic: the weights move away from 1
    assert opt.alph == pytest.approx(alpha, rel=1e-15)


# ----------------------------------------------------------------------------------------------- gossip ----
@pytest.mark.parametrize("graph", ["random_directed", "wheel", "star"])
def test_gossip_conserves_mass_and_debiasing_finds_the_average(graph):
    g = GRAPHS[graph][0]
    pr = LeastSquares([g], seed=4)
    opt = SGP(pr, "cpu", _conf(alpha0=0.0, outer_iterations=400))
    torch.manual_seed(3)
    x0 = torch.randn(pr.N, 5, dtype=torch.float64)
    opt.x[:, :5] = x0
    opt.arena.theta[:, :5] = x0
    avg = x0.mean(0)
    sum0 = opt.x.sum(0).clone()
    for _ in range(400):
        opt.run_rounds(1)
        assert (opt.x.sum(0) - sum0).abs().max().item() < 1e-13
        assert abs(opt.w.sum().item() - pr.N) < 1e-13
    th = opt.arena.theta[:, :5]
    err_theta = (th - avg).abs().max().item()
    err_x = (opt.x[:, :5] - avg).abs().max().item()
    print(f"\n{graph}: |theta - avg| {err_theta:.2e}, |x - avg| {err_x:.2e}, w in [{opt.w.min():.3f}, {opt.w.max():.3f}]")
    assert err_theta < 1e-12
    assert err_x > 1e-2            # x alone converges to the Perron-weighted average pi_i N avg


@pytest.mark.parametrize("graph", ["cycle6", "directed_cycle"])
def test_doubly_stochastic_graph_equals_dsgd(graph):
    """On the cycle push-sum weights are the Metropolis weights, w stays 1 and SGP is DSGD, up to rounding.  The
    directed cycle is doubly stochastic too (A = (I + P) / 2): SGP keeps w = 1 exactly there."""
    g = nx.cycle_graph(6) if graph == "cycle6" else GRAPHS["directed_cycle"][0]
    pr = LeastSquares([g], seed=5)
    s = SGP(pr, "cpu", _conf(mu=0.3, outer_iterations=300))
    s.run_rounds(300)
    assert torch.all(s.w == 1.0)
    if graph != "cycle6":
        return
    pr2 = LeastSquares([nx.cycle_graph(6)], seed=5)
    d = DSGD(pr2, "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.3, "outer_iterations": 300})
    d.run_rounds(300)
    a, b = s.arena.theta.numpy(), d.arena.theta.numpy()
    r = np.abs(a - b).max() / np.abs(b).max()
    print(f"\nsgp vs dsgd on the cycle: {r:.2e}")
    assert r < 1e-12


def test_heterogeneous_least_squares_reaches_the_dsgd_neighbourhood():
    """Node i minimises its own least-squares problem.  With a constant step, DSGD on the undirected cycle stops in an
    O(alpha) neighbourhood of the global minimiser; SGP on a random directed graph does the same: its distance shrinks
    with alpha as DSGD's does, is of DSGD's size, and is far below a node on its own."""
    g = GRAPHS["random_directed"][0]
    x_star = LeastSquares([g], seed=6).solution()

    def err(cls, graph, alpha):
        pr = LeastSquares([graph], seed=6)
        conf = {"alg_name": cls.alg_name, "alpha0": alpha, "mu": 0.0, "outer_iterations": 6000}
        o = cls(pr, "cpu", conf)
        o.run_rounds(6000)
        return np.abs(o.arena.theta.numpy()[:, :5] - x_star).max()

    e_sgp = {a: err(SGP, g, a) for a in (0.02, 0.005)}
    e_dsgd = {a: err(DSGD, nx.cycle_graph(7), a) for a in (0.02, 0.005)}
    pr = LeastSquares([g], seed=6)
    e_solo = np.abs(np.linalg.solve(pr.A[0].T @ pr.A[0], pr.A[0].T @ pr.b[0]) - x_star).max()
    print(f"\n|theta - x*|_max: sgp {e_sgp}, dsgd on the cycle {e_dsgd}, node 0 alone {e_solo:.3e}")
    for a in e_sgp:
        assert e_sgp[a] < 2.0 * e_dsgd[a] and e_sgp[a] < 0.2 * e_solo
    assert e_sgp[0.005] < 0.4 * e_sgp[0.02]


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["sgp"] is SGP
    base = {"alg_name": "sgp", "alpha0": 0.01, "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["mu"] == 0.0 and c["update_graph"] is True and c["profile"] is False
    for key in ("alpha0", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(base, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        SGP(LeastSquares([nx.cycle_graph(4)]), "cpu", _conf(mixing_order="reference"))


def _exp(graph_type, alg="sgp", **pc):
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"]["graph"] = {"type": graph_type, "num_nodes": 4, "p": 0.5, "gen_attempts": 50}
    p = conf["problem_configs"]["problem1"]
    p["optimizer_config"] = ({"alg_name": "sgp", "alpha0": 0.01, "outer_iterations": 3} if alg == "sgp" else
                             {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.0, "outer_iterations": 3})
    p.update(pc)
    return conf


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_needs_sgp_and_no_link_drop(graph_type):
    validate_experiment(_exp(graph_type), "mnist")
    with pytest.raises(ConfigError, match=r"experiment\.graph.*problem_configs\.problem1\.optimizer_config\.alg_name"):
        validate_experiment(_exp(graph_type, alg="dsgd"), "mnist")
    with pytest.raises(ConfigError, match=r"problem_configs\.problem1\.fault_injection"):
        validate_experiment(_exp(graph_type, fault_injection={"link_drop_prob": 0.2}), "mnist")
    # undirected graphs: SGP with fault injection, and the other algorithms, load as before
    validate_experiment(_exp("cycle", fault_injection={"link_drop_prob": 0.2}), "mnist")
    validate_experiment(_exp("cycle", alg="dsgd"), "mnist")


def test_directed_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_directed.yaml"), "mnist")
    assert conf["experiment"]["graph"] == {"type": "exponential", "num_nodes": 10}
    assert [p["optimizer_config"]["alg_name"] for p in conf["problem_configs"].values()] == ["sgp"]
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    for key in ("model", "data_split_type"):
        assert conf["experiment"][key] == paper["experiment"][key]


def test_link_drop_on_an_undirected_graph_runs():
    """Fault injection changes the graph every round; push-sum needs no rebuild of a doubly stochastic matrix."""
    conf = _conf(alpha0=0.02, outer_iterations=6)
    pr = _mnist_problem(conf)
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 1}
    pr._init_faults()
    opt = SGP(pr, "cpu", conf)
    opt.train()
    assert torch.isfinite(pr.arena.theta).all() and (opt.w > 0).all()
    assert torch.equal(pr.arena.theta, ref.sgp_debias(opt.x, opt.w))


# ------------------------------------------------------------------------------------------------ runner ----
def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch):
    from test_exact_diffusion import _synthetic
    dist_mnist_ex = _synthetic(monkeypatch)
    conf = _exp("exponential")
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="sgp")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "sgp", "alpha0": 0.01, "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    assert {"graph.gpickle", "sgp_results.pt"} <= set(os.listdir(outs[0]))
    res = torch.load(os.path.join(outs[0], "sgp_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"}
    assert len(res["validation_loss"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def _mnist_problem(conf, N=4, M=100, graph=None):
    from test_exact_diffusion import _mnist_problem as mk
    pr = mk(conf, N=N, M=M)
    if graph is not None:
        pr.graph = pr._base_graph = graph
    return pr


def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, outer_iterations=6)
    g = nx.DiGraph([(0, 1), (1, 2), (2, 3), (3, 0), (0, 2)])
    full = _mnist_problem(conf, graph=g)
    of = SGP(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf, graph=g)
    o1 = SGP(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3 and not torch.all(o1.w == 1.0)
    second = _mnist_problem(conf, graph=g)
    o2 = SGP(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.x, o1.x) and torch.equal(o2.w, o1.w)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.x, of.x) and torch.equal(o2.w, of.w)
    assert o2.alph == of.alph
    assert second.forward_cnt == full.forward_cnt
