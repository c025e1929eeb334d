"""Push-DIGing (gradient tracking on push-sum gossip) on the PyTorch path (CPU): a float64 oracle round by round on
directed, irregular undirected and changing graphs, the tracking and push-sum invariants, DSGT equivalence on the
cycle, exactness on a heterogeneous problem where SGP is biased, configuration, the MNIST runner and
checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import push_diging_oracle as po
from test_exact_diffusion import LeastSquares
from test_sgp import GRAPHS, _gen
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGT, SGP, PushDIGing
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


# three strongly connected digraphs on 7 nodes, one after the other every round
SWITCH3 = [_gen("directed_cycle", 7), _gen("exponential", 7), _gen("random_directed", 7, p=0.3, seed=4, gen_attempts=200)]
TRACK_GRAPHS = {"random_directed": GRAPHS["random_directed"], "star": GRAPHS["star"], "switch3": SWITCH3}


def _conf(**kw):
    return dict({"alg_name": "push_diging", "alpha": 0.05, "outer_iterations": 50}, **kw)


def _np(t):
    return t.double().numpy()[:, :5].copy()


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph):
    gs = GRAPHS[graph]
    pr = LeastSquares(gs, seed=1)
    opt = PushDIGing(pr, "cpu", _conf())
    u, y, g = _np(opt.u), np.zeros((pr.N, 5)), np.zeros((pr.N, 5))
    w = np.ones(pr.N)
    for k in range(12):
        gr = gs[(pr.idx + 1) % len(gs)]          # the round refreshes the graph first
        opt.run_rounds(1)
        u, w, y, g, th = po.pdg_round(u, w, y, g, gr, pr.grad, 0.05)
        np.testing.assert_allclose(_np(opt.u), u, rtol=1e-12, atol=1e-13, err_msg=f"round {k} u")
        np.testing.assert_allclose(opt.w.numpy(), w, rtol=1e-14, atol=0, err_msg=f"round {k} w")
        np.testing.assert_allclose(_np(opt.y), y, rtol=1e-12, atol=1e-13, err_msg=f"round {k} y")
        np.testing.assert_allclose(_np(opt.g), g, rtol=1e-12, atol=1e-13, err_msg=f"round {k} g_old")
        np.testing.assert_allclose(_np(opt.arena.theta), th, rtol=1e-12, atol=1e-13, err_msg=f"round {k} theta")
    if graph in ("wheel", "star", "random_directed"):
        assert np.abs(w - 1.0).max() > 1e-2          # not doubly stochastic: the weights move away from 1


@pytest.mark.parametrize("graph", sorted(TRACK_GRAPHS))
def test_tracking_and_push_sum_invariants_every_round(graph):
    """A column-stochastic A preserves sums: sum y = sum g (the tracker follows the network gradient), sum w = N, and
    the mix moves sum u by exactly -alpha sum y."""
    gs = TRACK_GRAPHS[graph]
    pr = LeastSquares(gs, seed=2)
    alpha = 0.03
    opt = PushDIGing(pr, "cpu", _conf(alpha=alpha, outer_iterations=300))
    for k in range(300):
        su, sy = opt.u.sum(0).clone(), opt.y.sum(0).clone()
        opt.run_rounds(1)
        scale = 1.0 + opt.g.abs().sum(0).max().item()
        assert (opt.y.sum(0) - opt.g.sum(0)).abs().max().item() < 1e-13 * scale, k
        assert abs(opt.w.sum().item() - pr.N) < 1e-13, k
        assert (opt.u.sum(0) - (su - alpha * sy)).abs().max().item() < 1e-12 * (1.0 + su.abs().max().item()), k


def test_undirected_cycle_equals_dsgt_without_init_grads_and_directed_cycle_keeps_w_1():
    """On the cycle the push weights are the Metropolis weights, w stays 1 and Push-DIGing is DSGT with
    ``init_grads: false``, up to rounding.  The directed cycle is doubly stochastic too: w = 1 exactly."""
    pr = LeastSquares([nx.cycle_graph(6)], seed=5)
    p = PushDIGing(pr, "cpu", _conf(outer_iterations=300))
    p.run_rounds(300)
    assert torch.all(p.w == 1.0)
    pr2 = LeastSquares([nx.cycle_graph(6)], seed=5)
    d = DSGT(pr2, "cpu", {"alg_name": "dsgt", "alpha": 0.05, "init_grads": False, "outer_iterations": 300})
    d.run_rounds(300)
    # y tends to 0 with the network gradient: its rounding is measured against the size of the local gradients
    for name, a, b, scale in (("theta", p.arena.theta, d.arena.theta, d.arena.theta), ("y", p.y, d.y, d.g)):
        r = ((a - b).abs().max() / scale.abs().max()).item()
        print(f"\npush_diging vs dsgt on the cycle, {name}: {r:.2e}")
        assert r < 1e-12, name
    pr3 = LeastSquares(GRAPHS["directed_cycle"], seed=5)
    q = PushDIGing(pr3, "cpu", _conf(outer_iterations=300))
    q.run_rounds(300)
    assert torch.all(q.w == 1.0)


@pytest.mark.parametrize("graph", ["random_directed", "switch3"])
def test_heterogeneous_least_squares_is_exact_where_sgp_is_biased(graph):
    """Node i minimises its own least-squares problem.  With a constant step SGP stops in an O(alpha) neighbourhood of
    the global minimiser; gradient tracking removes that bias and reaches x* to round-off, on a fixed random digraph
    and on three digraphs taking turns every round."""
    gs = TRACK_GRAPHS[graph]
    x_star = LeastSquares(gs, seed=6).solution()

    def err(cls, conf):
        o = cls(LeastSquares(gs, seed=6), "cpu", dict(conf, outer_iterations=6000))
        o.run_rounds(6000)
        return np.abs(o.arena.theta.numpy()[:, :5] - x_star).max()

    e_pdg = err(PushDIGing, _conf(alpha=0.02))
    e_sgp = err(SGP, {"alg_name": "sgp", "alpha0": 0.02, "mu": 0.0})
    print(f"\n{graph}: |theta - x*|_max push_diging {e_pdg:.2e}, sgp {e_sgp:.2e}")
    assert e_pdg < 1e-9
    assert e_sgp > 1e-2


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["push_diging"] is PushDIGing
    base = {"alg_name": "push_diging", "alpha": 0.01, "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["update_graph"] is True and c["profile"] is False
    assert "init_grads" not in c and "mu" not in c
    for key in ("alpha", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(base, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        PushDIGing(LeastSquares([nx.cycle_graph(4)]), "cpu", _conf(mixing_order="reference"))


def _exp(graph_type, alg="push_diging", **pc):
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"]["graph"] = {"type": graph_type, "num_nodes": 4, "p": 0.5, "gen_attempts": 50}
    p = conf["problem_configs"]["problem1"]
    p["optimizer_config"] = ({"alg_name": "push_diging", "alpha": 0.01, "outer_iterations": 3} if alg == "push_diging"
                             else {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.0, "outer_iterations": 3})
    p.update(pc)
    return conf


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_runs_push_diging_and_refuses_dsgd_and_link_drop(graph_type):
    validate_experiment(_exp(graph_type), "mnist")
    with pytest.raises(ConfigError, match=r"experiment\.graph.*sgp or push_diging.*problem_configs\.problem1\."
                                          r"optimizer_config\.alg_name"):
        validate_experiment(_exp(graph_type, alg="dsgd"), "mnist")
    with pytest.raises(ConfigError, match=r"problem_configs\.problem1\.fault_injection"):
        validate_experiment(_exp(graph_type, fault_injection={"link_drop_prob": 0.2}), "mnist")
    validate_experiment(_exp("cycle", fault_injection={"link_drop_prob": 0.2}), "mnist")


def test_link_drop_on_a_directed_graph_is_refused_by_the_optimizer():
    conf = _conf(alpha=0.02, outer_iterations=3)
    pr = _mnist_problem(conf, graph=nx.DiGraph([(0, 1), (1, 2), (2, 3), (3, 0)]))
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 1}
    with pytest.raises(ValueError, match="fault_injection"):
        PushDIGing(pr, "cpu", conf)


def test_directed_tracking_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_directed_tracking.yaml"), "mnist")
    assert conf["experiment"]["graph"] == {"type": "exponential", "num_nodes": 10}
    opts = {p["optimizer_config"]["alg_name"]: p["optimizer_config"] for p in conf["problem_configs"].values()}
    assert set(opts) == {"push_diging", "sgp"}
    assert opts["push_diging"]["alpha"] == 0.005
    directed = load_experiment(os.path.join(EXP, "dist_mnist_directed.yaml"), "mnist")
    for key in ("model", "data_split_type", "graph", "data_source"):
        assert conf["experiment"].get(key) == directed["experiment"].get(key), key
    assert opts["sgp"] == next(iter(directed["problem_configs"].values()))["optimizer_config"]


# ------------------------------------------------------------------------------------------------ runner ----
def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch):
    from test_exact_diffusion import _synthetic
    dist_mnist_ex = _synthetic(monkeypatch)
    conf = _exp("exponential")
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="push_diging")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "push_diging", "alpha": 0.01, "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    assert {"graph.gpickle", "push_diging_results.pt"} <= set(os.listdir(outs[0]))
    res = torch.load(os.path.join(outs[0], "push_diging_results.pt"), weights_only=False)
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
    conf = _conf(alpha=0.02, outer_iterations=6)
    g = nx.DiGraph([(0, 1), (1, 2), (2, 3), (3, 0), (0, 2)])
    full = _mnist_problem(conf, graph=g)
    of = PushDIGing(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf, graph=g)
    o1 = PushDIGing(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3 and not torch.all(o1.w == 1.0) and o1.y.abs().max() > 0
    second = _mnist_problem(conf, graph=g)
    o2 = PushDIGing(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3
    for name in ("u", "w", "y", "g"):
        assert torch.equal(getattr(o2, name), getattr(o1, name)), name
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in ("u", "w", "y", "g"):
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt
