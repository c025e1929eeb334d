"""BRIDGE on the PyTorch path (CPU): the float64 oracle round by round with and without attackers, the screening
guarantee, neighbor-order independence, robustness on least squares with one shared minimiser, configuration, the yaml,
both runners, checkpoint/resume with an ALIE attacker and the fused mix's neighbor capacity."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import bridge_oracle as bo
from test_clipped_gossip import SharedMinimiser
from test_exact_diffusion import GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, Bridge, ClippedGossip
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")

# Byzantine sets per graph: adjacent attackers (0, 1 on the cycle and the complete graph), an honest node whose only
# neighbor attacks (node 5 of the isolated graph), an isolated attacker (6)
BYZ = {"cycle": [0, 1], "wheel": [0, 3], "complete": [0, 1], "random": [2], "isolated": [4, 6], "switching": [1]}
SCREENS = [("trimmed_mean", 0), ("trimmed_mean", 1), ("trimmed_mean", 2), ("median", None)]


def _conf(screen="trimmed_mean", b=1, **kw):
    c = {"alg_name": "bridge", "alpha0": 0.05, "mu": 0.0, "screen": screen, "outer_iterations": 50}
    if screen == "trimmed_mean":
        c["b"] = b
    return dict(c, **kw)


def _np(t, n=5):
    return t[:, :n].double().numpy().copy()


def _attack(byz, attack):
    return {i: bo.ATTACK[attack] for i in byz} if attack else {}


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("attack", [None, "sign_flip", "alie"])
@pytest.mark.parametrize("screen,b", SCREENS)
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "isolated", "switching"])
def test_torch_path_matches_float64_oracle_round_by_round(graph, screen, b, attack):
    pr = LeastSquares(GRAPHS[graph], seed=1)
    byz = BYZ[graph] if attack else []
    conf = _conf(screen, b)
    if attack:
        conf["byzantine"] = {"nodes": byz, "attack": attack, "scale": 2.0, "z": 1.5}
    opt = Bridge(pr, "cpu", conf)
    theta = _np(opt.arena.theta)
    pub = theta.copy()
    for k in range(8):
        opt.run_rounds(1)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        theta, pub, _ = bo.round_(theta, pub, W, pr.grad, 0.05, screen, b or 0, _attack(byz, attack), 2.0, 1.5)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        np.testing.assert_allclose(_np(opt.pub), pub, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")


@pytest.mark.parametrize("screen,b", SCREENS)
def test_link_drops_match_the_oracle_on_the_dropped_graphs(screen, b):
    conf = _conf(screen, b, alpha0=0.02, outer_iterations=6, byzantine={"nodes": [1], "attack": "alie", "z": 1.0})
    pr = _mnist_problem(conf)
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 6}
    pr._init_faults()
    opt = Bridge(pr, "cpu", copy.deepcopy(conf))
    n = pr.layout.n
    graphs = set()
    for k in range(6):
        theta0, pub0 = _np(pr.arena.theta, n), _np(opt.pub, n)
        opt.run_rounds(1)
        W = pr.topology().W
        graphs.add(W.tobytes())
        mixed = bo.mix(theta0, pub0, W, screen, b or 0)
        # the step is theta - alpha g: the mixed rows are recovered from theta + alpha g
        got = _np(pr.arena.theta, n) + opt.alph * _np(pr.arena.grad, n)
        np.testing.assert_allclose(got, mixed, rtol=0, atol=1e-5, err_msg=f"round {k}")
    assert len(graphs) > 2


# --------------------------------------------------------------------------------------------- guarantee ----
@pytest.mark.parametrize("attack", ["sign_flip", "alie"])
@pytest.mark.parametrize("screen,b", SCREENS)
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "isolated", "switching"])
def test_screening_guarantee_every_round(graph, screen, b, attack):
    """An honest node with at most b Byzantine neighbors (trimmed mean), or with fewer Byzantine than honest values in
    its set (median), lands inside [min, max] of its own and its honest neighbors' values, element by element."""
    pr = LeastSquares(GRAPHS[graph], seed=5)
    byz = set(BYZ[graph])
    conf = _conf(screen, b, byzantine={"nodes": sorted(byz), "attack": attack, "scale": 4.0, "z": 3.0})
    opt = Bridge(pr, "cpu", conf)
    for k in range(10):
        theta0, pub0 = _np(opt.arena.theta), _np(opt.pub)
        opt.run_rounds(1)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        mixed = _np(opt.arena.theta) + opt.alph * _np(opt.arena.grad)
        for i in range(pr.N):
            if bo.guaranteed(W, i, byz, screen, b or 0):
                lo, hi = bo.honest_range(theta0, pub0, W, i, byz)
                slack = 1e-12 * (1 + np.abs(lo) + np.abs(hi))
                assert np.all(mixed[i] >= lo - slack) and np.all(mixed[i] <= hi + slack), f"round {k} node {i}"


@pytest.mark.parametrize("screen,b", SCREENS)
def test_result_does_not_depend_on_neighbor_order(screen, b):
    rng = np.random.default_rng(7)
    x = rng.standard_normal(64)
    vals = rng.standard_normal((9, 64))
    vals[3] = vals[5]                                       # ties
    want = torch.tensor(bo.screen(x, vals, screen, b or 0))
    for seed in range(6):
        perm = np.random.default_rng(seed).permutation(9)
        theta = torch.tensor(x[None, :])
        pub_all = torch.tensor(np.vstack([x[None, :], vals[perm]]))
        ref.bridge_mix_(theta, pub_all, [list(range(1, 10))], 0, screen, b or 0)
        assert torch.equal(theta[0], want), f"permutation {perm}"


def test_node_with_deg_at_most_2b_keeps_its_row():
    g = nx.star_graph(5)                                    # hub degree 5, leaves degree 1
    theta = torch.randn(6, 7, dtype=torch.float64)
    theta0 = theta.clone()
    ref.bridge_mix_(theta, -7.0 * theta, [sorted(g.neighbors(i)) for i in range(6)], 0, "trimmed_mean", 3)
    assert torch.equal(theta, theta0)
    x = np.arange(4.0)
    assert np.array_equal(bo.screen(x, np.zeros((4, 4)), "trimmed_mean", 2), x)


def test_trimmed_mean_b0_is_the_unweighted_neighborhood_mean():
    rng = np.random.default_rng(1)
    x, vals = rng.standard_normal(8), rng.standard_normal((3, 8))
    np.testing.assert_allclose(bo.screen(x, vals, "trimmed_mean", 0), (x + vals.sum(0)) / 4, rtol=1e-15)


# --------------------------------------------------------------------------------------------- robustness ----
@pytest.mark.parametrize("attack,scale,z", [("sign_flip", 10.0, 1.0), ("alie", 1.0, 10.0)])
def test_screens_keep_the_honest_nodes_at_the_minimiser(attack, scale, z):
    """10-node complete graph, nodes 0 and 1 attack: every honest node has 9 neighbors, 2 Byzantine.  Without a defence
    the honest nodes end far from x*; both screens end at x*.  Distances after 600 rounds on the float64 CPU path
    (seed 0): sign flip (scale 10) 5.6e15 without a defence, 1.8e-8 with the trimmed mean (b 2) and 4.8e-9 with the
    median; ALIE (z 10) 3.3 without, 1.4e-10 and 8.6e-11."""
    R, err = 600, {}
    byz = {"nodes": [0, 1], "attack": attack, "scale": scale, "z": z}
    arms = {"none": (ClippedGossip, {"alg_name": "clipped_gossip", "alpha0": 0.05, "clip": "none"}),
            "trimmed_mean": (Bridge, _conf("trimmed_mean", 2)), "median": (Bridge, _conf("median"))}
    for name, (cls, conf) in arms.items():
        pr = SharedMinimiser([nx.complete_graph(10)], seed=0)
        opt = cls(pr, "cpu", dict(conf, outer_iterations=R, byzantine=byz))
        opt.run_rounds(R)
        th = _np(opt.arena.theta)[2:]
        err[name] = np.abs(th - pr.x_star).max() if np.isfinite(th).all() else np.inf
    print(f"\n{attack}: max |theta_honest - x*| " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert err["none"] > 1.0
    assert err["trimmed_mean"] < 1e-7 and err["median"] < 1e-7


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_refusals():
    assert ALGORITHMS["bridge"] is Bridge
    base = {"alg_name": "bridge", "alpha0": 0.01, "screen": "trimmed_mean", "b": 1, "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["mu"] == 0.0 and c["update_graph"] is True and "byzantine" not in c
    for key in ("alpha0", "screen", "outer_iterations", "b"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    med = {k: v for k, v in base.items() if k != "b"}
    validate_optimizer(dict(med, screen="median"))
    with pytest.raises(ConfigError, match="b applies to screen trimmed_mean only"):
        validate_optimizer(dict(base, screen="median"))
    with pytest.raises(ConfigError, match="screen must be one of trimmed_mean|median"):
        validate_optimizer(dict(base, screen="krum"))
    for b in (True, 1.0, "1", -1):
        with pytest.raises(ConfigError, match="b must be an integer >= 0"):
            validate_optimizer(dict(base, b=b))
    validate_optimizer(dict(base, b=0))
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(base, mixing_order="reference"))
    byz = {"nodes": [0], "attack": "alie", "z": 2.0}
    validate_optimizer(dict(base, byzantine=byz))
    with pytest.raises(ConfigError, match="attack must be one of"):
        validate_optimizer(dict(base, byzantine=dict(byz, attack="label_flip")))
    with pytest.raises(ConfigError, match=r"byzantine.*clipped_gossip only.*bridge.*'relaysum'"):
        validate_optimizer({"alg_name": "relaysum", "alpha0": 0.1, "mu": 0.0, "outer_iterations": 3,
                            "byzantine": byz})
    conf = _exp("cycle")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(base, byzantine=dict(byz, nodes=[4]))
    with pytest.raises(ConfigError, match="out of range"):
        validate_experiment(copy.deepcopy(conf), "mnist")
    pr = LeastSquares(GRAPHS["cycle"])
    with pytest.raises(ValueError, match="screen must be one of"):
        Bridge(pr, "cpu", _conf("mean"))
    with pytest.raises(ValueError, match="b must be an integer"):
        Bridge(pr, "cpu", _conf("trimmed_mean", -2))
    with pytest.raises(ValueError, match="jacobi"):
        Bridge(pr, "cpu", _conf(mixing_order="reference"))
    with pytest.raises(ValueError, match="undirected"):
        Bridge(LeastSquares([nx.cycle_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = {"alg_name": "bridge", "alpha0": 0.01,
                                                               "screen": "median", "outer_iterations": 3}
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'bridge'"):
        validate_experiment(conf, "mnist")


def test_fused_mix_refuses_more_neighbors_than_its_registers_hold():
    from nn_distributed_training_b200.ops.engine import BRIDGE_MAX_DEG, check_bridge_capacity
    check_bridge_capacity(BRIDGE_MAX_DEG)
    with pytest.raises(ValueError, match=f"at most {BRIDGE_MAX_DEG} neighbors per node.*a node with 17"):
        check_bridge_capacity(17)


def test_bridge_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_bridge.yaml"), "mnist")
    assert conf["experiment"]["graph"] == {"num_nodes": 10, "type": "complete"}
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    arms = [(o["alg_name"], o.get("clip"), o.get("screen"), o["byzantine"]["attack"]) for o in ocs]
    want = []
    for attack in ("sign_flip", "alie"):
        want += [("clipped_gossip", "none", None, attack), ("clipped_gossip", "adaptive", None, attack),
                 ("bridge", None, "trimmed_mean", attack), ("bridge", None, "median", attack)]
    assert arms == want
    for o in ocs:
        assert o["complete_graph_mode"] == "pointer" and o["byzantine"]["nodes"] == [0, 1]
        if o.get("clip") == "adaptive":
            assert o["delta"] == 0.2
        if o.get("screen") == "trimmed_mean":
            assert o["b"] == 2


# ------------------------------------------------------------------------------------------------ runners ----
def test_mnist_runner_writes_byzantine_nodes(tmp_path, monkeypatch):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_bridge.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True, use_cuda=False)
    conf["experiment"]["graph"]["num_nodes"] = 5
    conf["problem_configs"] = {k: v for k, v in conf["problem_configs"].items()
                               if v["optimizer_config"]["alg_name"] == "bridge"}
    for pc in conf["problem_configs"].values():
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"]["outer_iterations"] = 3
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_bridge"))
    assert len(out) == 1
    for pc in conf["problem_configs"].values():
        res = torch.load(os.path.join(out[0], f"{pc['problem_name']}_results.pt"), weights_only=False)
        assert res["byzantine_nodes"] == [0, 1]
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])


def test_density_runner_runs_bridge(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="br")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "bridge", "alpha0": 0.01, "screen": "median", "outer_iterations": 4,
                              "byzantine": {"nodes": [2], "attack": "sign_flip"}}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "br_results.pt"), weights_only=False)
    assert res["byzantine_nodes"] == [2]
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("screen,b", [("trimmed_mean", 1), ("median", None)])
def test_checkpoint_resume_with_an_alie_attacker_is_bit_exact(tmp_path, screen, b):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(screen, b, alpha0=0.02, outer_iterations=6, byzantine={"nodes": [1], "attack": "alie", "z": 1.0})
    full = _mnist_problem(conf)
    of = Bridge(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = Bridge(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    second = _mnist_problem(conf)
    o2 = Bridge(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.pub, o1.pub)
    assert not torch.equal(o2.pub[1], second.arena.theta[1])      # the ALIE row is not the attacker's theta
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.pub, of.pub)
