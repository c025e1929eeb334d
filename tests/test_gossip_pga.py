"""Gossip-PGA and local SGD on the PyTorch path (CPU, float64): the NumPy oracle round by round on six graph kinds at
periods 1, 2, 3 and 5 with and without link drops and gossip, equal rows after every global round and the node mean
kept by both mixes, DSGD at a period past the run bit for bit, DSGD on the complete graph at period 1, local SGD without
averaging as N separate SGD runs, exactness on heterogeneous least squares at period 1, every configuration refusal,
the runners and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import pga_oracle as po
from hsgd_oracle import metropolis
from test_exact_diffusion import _mnist_problem, _synthetic
from test_gt_hsgd import GRAPHS, LSProblem, _np
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, GossipPGA
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
PERIODS = [1, 2, 3, 5]
DROPS = {"link_drop_prob": 0.3, "seed": 5, "from_round": 2, "to_round": 12}


def _conf(**kw):
    return dict({"alg_name": "gossip_pga", "alpha0": 0.05, "mu": 0.5, "period": 3, "outer_iterations": 50}, **kw)


def _alphas(alpha0, mu, n):
    out, a = [], alpha0
    for _ in range(n):
        a = a * (1.0 - mu * a)
        out.append(a)
    return out


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])
@pytest.mark.parametrize("drops", [False, True], ids=["static", "link_drops"])
@pytest.mark.parametrize("period", PERIODS)
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph, period, drops, gossip):
    R = 12
    pr = LSProblem(GRAPHS[graph], batch=8, seed=1, faults=DROPS if drops else None)
    Ws = [metropolis(g) for g in pr.plan_graphs(R, 0, 1)]
    if drops:
        assert any(not np.array_equal(W, Ws[0]) for W in Ws)
    opt = GossipPGA(pr, "cpu", _conf(period=period, gossip=gossip, outer_iterations=R))
    want = po.run(_np(pr.arena.theta), Ws, _alphas(0.05, 0.5, R), period, gossip, pr.batch_grad, R)
    for k, theta in enumerate(want):
        opt.run_rounds(1)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-11, atol=1e-11, err_msg=f"round {k}")
    assert pr.calls.tolist() == [R] * pr.N
    assert opt.alph == _alphas(0.05, 0.5, R)[-1]


@pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])
@pytest.mark.parametrize("graph", ["cycle", "star", "random"])
def test_rows_equal_after_every_global_round_and_both_mixes_keep_the_mean(graph, gossip):
    """With alpha0 = 0 a round is its mix alone: after a global round every row is the same bit for bit, and every round
    keeps the node mean to round-off (W is doubly stochastic; the global mean is the mean)."""
    pr = LSProblem(GRAPHS[graph], batch=8, seed=2, faults=DROPS)
    pr.arena.theta[:, :5] = torch.as_tensor(np.random.default_rng(0).standard_normal((pr.N, 5)))
    opt = GossipPGA(pr, "cpu", _conf(alpha0=0.0, period=3, gossip=gossip, outer_iterations=12))
    mean0 = _np(pr.arena.theta).mean(0)
    for k in range(12):
        opt.run_rounds(1)
        th = _np(pr.arena.theta)
        np.testing.assert_allclose(th.mean(0), mean0, rtol=0, atol=1e-14 * np.abs(mean0).max(), err_msg=f"round {k}")
        if opt.is_global(k):
            assert (th == th[0]).all(), f"round {k}"
        elif k < 2:                                             # round 2 is the first global one
            assert not (th == th[0]).all(), f"round {k}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_pga_mean_is_the_float64_mean_cast_once(dtype):
    g = torch.Generator().manual_seed(0)
    rows = torch.randn(7, 33, generator=g, dtype=torch.float64).to(dtype)
    out = torch.empty(3, 33, dtype=dtype)
    ref.pga_mean_(out, rows)
    s = np.zeros(33)
    for j in range(7):
        s = s + rows[j].double().numpy()
    want = torch.as_tensor(s / 7).to(dtype)
    assert all(torch.equal(out[i], want) for i in range(3))


# ------------------------------------------------------------------------------------------ equivalences ----
@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_period_past_the_run_is_dsgd_bit_for_bit(model):
    R = 10
    pconf = _conf(period=R + 1, outer_iterations=R)
    dconf = {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": R}
    if model == "mnist":
        pa, pb = _mnist_problem(pconf), _mnist_problem(dconf)
    else:
        pa, pb = (LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS),
                  LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS))
    a, b = GossipPGA(pa, "cpu", pconf), DSGD(pb, "cpu", dconf)
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"
        assert a.alph == b.alph
    assert pa.forward_cnt == pb.forward_cnt and (pa.calls == pb.calls).all()


@pytest.mark.parametrize("graph", ["cycle", "path", "star"])
def test_period_one_is_dsgd_on_the_complete_graph(graph):
    """period 1 averages every round: DSGD on the complete graph (W = 11^T / N), to round-off."""
    R = 10
    N = GRAPHS[graph].number_of_nodes()
    pa = LSProblem(GRAPHS[graph], batch=8, seed=3)
    pb = LSProblem(nx.complete_graph(N), batch=8, seed=3)
    pb.arena.theta.copy_(pa.arena.theta)
    a = GossipPGA(pa, "cpu", _conf(period=1, outer_iterations=R))
    b = DSGD(pb, "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": R})
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        np.testing.assert_allclose(_np(pa.arena.theta), _np(pb.arena.theta), rtol=1e-13, atol=1e-13, err_msg=f"{k}")


def test_local_sgd_without_averaging_is_n_separate_sgd_runs():
    """gossip: false and period > outer_iterations: no node ever reads another, each follows its own SGD trajectory."""
    R = 10
    pr = LSProblem(GRAPHS["wheel"], batch=8, seed=4)
    theta = _np(pr.arena.theta)
    opt = GossipPGA(pr, "cpu", _conf(period=R + 1, gossip=False, outer_iterations=R))
    for k, a in enumerate(_alphas(0.05, 0.5, R)):
        opt.run_rounds(1)
        theta = theta - a * pr.batch_grad(theta, k)
        np.testing.assert_allclose(_np(pr.arena.theta), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")


def test_period_one_reaches_the_least_squares_minimiser_where_dsgd_does_not():
    """Heterogeneous least squares, full-batch gradients, cycle, constant step: at period 1 the row mean is gradient
    descent on sum_i f_i and converges to its minimiser; DSGD stops a measurable distance away."""
    rounds, alpha = 2000, 0.02
    pr = LSProblem(nx.cycle_graph(8), seed=3)
    opt = GossipPGA(pr, "cpu", _conf(alpha0=alpha, mu=0.0, period=1, outer_iterations=rounds))
    opt.run_rounds(rounds)
    err = np.abs(_np(opt.arena.theta).mean(0) - pr.solution()).max()
    pd = LSProblem(nx.cycle_graph(8), seed=3)
    od = DSGD(pd, "cpu", {"alg_name": "dsgd", "alpha0": alpha, "mu": 0.0, "outer_iterations": rounds})
    od.run_rounds(rounds)
    err_dsgd = np.abs(_np(od.arena.theta).mean(0) - pd.solution()).max()
    print(f"\nmax |mean theta - x*| Gossip-PGA (period 1) {err:.2e}, DSGD {err_dsgd:.2e}")
    assert err < 1e-9
    assert err_dsgd > 1e-3


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "gossip_pga", "alpha0": 0.01, "period": 4, "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["gossip_pga"] is GossipPGA
    c = validate_optimizer(dict(BASE))
    assert c["mu"] == 0.0 and c["gossip"] is True and c["update_graph"] is True and c["profile"] is False
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, alpha0=0.0, mu=0.1, period=1, gossip=False, update_graph=False, profile=True))


@pytest.mark.parametrize("key", ["alpha0", "period", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})


@pytest.mark.parametrize("alpha0", [-0.1, float("inf"), float("nan"), "0.1", True])
def test_alpha0_must_be_finite_and_nonnegative(alpha0):
    with pytest.raises(ConfigError, match="alpha0"):
        validate_optimizer(dict(BASE, alpha0=alpha0))
    if not isinstance(alpha0, (str, bool)):
        with pytest.raises(ValueError, match="alpha0"):
            GossipPGA(LSProblem(GRAPHS["cycle"]), "cpu", _conf(alpha0=alpha0))


@pytest.mark.parametrize("period", [0, -2, 2.0, 1.5, "3", True, False])
def test_period_must_be_an_integer_of_at_least_one(period):
    with pytest.raises(ConfigError, match="period"):
        validate_optimizer(dict(BASE, period=period))
    with pytest.raises(ValueError, match="period"):
        GossipPGA(LSProblem(GRAPHS["cycle"]), "cpu", _conf(period=period))


@pytest.mark.parametrize("gossip", [1, 0, "true", None])
def test_gossip_must_be_a_bool(gossip):
    with pytest.raises(ConfigError, match="gossip"):
        validate_optimizer(dict(BASE, gossip=gossip))
    with pytest.raises(ValueError, match="gossip"):
        GossipPGA(LSProblem(GRAPHS["cycle"]), "cpu", _conf(gossip=gossip))


@pytest.mark.parametrize("key", ["alpha", "beta", "local_steps", "gossip_steps"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"gossip_pga takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        GossipPGA(LSProblem(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        GossipPGA(LSProblem(GRAPHS["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'gossip_pga'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        GossipPGA(LSProblem(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())


def test_changing_graphs_and_link_drops_are_accepted():
    pr = LSProblem(GRAPHS["cycle"], faults=dict(DROPS, from_round=0, to_round=6))
    assert len({tuple(sorted(g.edges())) for g in pr.plan_graphs(6, 0, 1)}) > 1
    GossipPGA(pr, "cpu", _conf(outer_iterations=6)).run_rounds(6)
    assert np.isfinite(pr.arena.theta.numpy()).all()


# ------------------------------------------------------------------------------------------------ runners ----
ARMS = [("dsgd", None, None), ("dsgt", None, None), ("gossip_pga", 4, True), ("gossip_pga", 16, True),
        ("gossip_pga", 4, False)]
NAMES = ["dsgd", "dsgt", "gossip_pga_p4", "gossip_pga_p16", "local_sgd_p4"]


def test_pga_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_pga.yaml"), "mnist")
    pcs = list(conf["problem_configs"].values())
    ocs = [p["optimizer_config"] for p in pcs]
    assert [(o["alg_name"], o.get("period"), o.get("gossip")) for o in ocs] == ARMS
    assert [p["problem_name"] for p in pcs] == NAMES
    assert all(p["train_batch_size"] == 64 for p in pcs)
    assert all(o.get("alpha0", o.get("alpha")) == 0.005 for o in ocs)
    e = conf["experiment"]
    assert e["graph"]["type"] == "cycle" and e["graph"]["num_nodes"] == 10 and e["data_split_type"] == "hetero"


def test_mnist_runner_on_the_pga_yaml(tmp_path, monkeypatch):
    """The five problems of the YAML at a tiny size; DSGD and every Gossip-PGA arm draw one batch per round."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_pga.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True, use_cuda=False)
    conf["experiment"]["graph"]["num_nodes"] = 4
    for pc in conf["problem_configs"].values():
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"]["outer_iterations"] = 5
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_pga"))
    assert len(out) == 1
    fp = {}
    for name in NAMES:
        res = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])
        fp[name] = [int(torch.as_tensor(v).sum()) for v in res["forward_pass_count"]]
    del fp["dsgt"]                   # init_grads: true draws one batch more
    assert len({tuple(v) for v in fp.values()}) == 1


def test_density_runner_runs_gossip_pga(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="gossip_pga")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "gossip_pga", "alpha0": 0.01, "period": 2, "outer_iterations": 4}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "gossip_pga_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("stop", [3, 5], ids=["odd_round", "before_global_round"])
def test_checkpoint_resume_is_bit_exact(tmp_path, stop):
    """period 3: round 5 is global, so stopping after 5 rounds resumes just before a global round; 3 is odd."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, period=3, outer_iterations=8)
    assert GossipPGA(_mnist_problem(conf), "cpu", copy.deepcopy(conf)).is_global(5)
    full = _mnist_problem(conf)
    of = GossipPGA(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = GossipPGA(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=stop, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = stop                   # "crash" after round `stop`
    o1.train()
    assert o1.k == stop
    second = _mnist_problem(conf)
    o2 = GossipPGA(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=stop, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == stop and o2.alph == o1.alph
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert o2.alph == of.alph
    assert second.forward_cnt == full.forward_cnt
