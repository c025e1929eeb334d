"""ClippedGossip on the PyTorch path (CPU): the float64 oracle round by round with and without attackers, the clipping
invariants, DSGD equivalences, robustness on least squares with one shared minimiser, configuration, the MNIST runner's
``byzantine_nodes``, the honest-only summary and checkpoint/resume with an ALIE attacker."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import clipped_gossip_oracle as co
from test_exact_diffusion import GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, ClippedGossip
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


def _conf(**kw):
    return dict({"alg_name": "clipped_gossip", "alpha0": 0.05, "mu": 0.0, "clip": "adaptive", "delta": 0.3,
                 "outer_iterations": 50}, **kw)


def _np(t, n=5):
    return t[:, :n].double().numpy().copy()


def _attack(byz, attack):
    return {i: co.ATTACK[attack] for i in byz} if attack else {}


# Byzantine sets per graph: adjacent attackers (0, 1 on the cycle and the complete graph), an honest node whose
# neighbors are all Byzantine (node 5 of the isolated graph: its one neighbor 4 attacks), an isolated attacker (6)
BYZ = {"cycle": [0, 1], "wheel": [0, 3], "complete": [0, 1], "random": [2], "isolated": [4, 6], "switching": [1]}
DELTAS = [0.0, 0.15, 0.3, 0.45]


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("attack", [None, "sign_flip", "alie"])
@pytest.mark.parametrize("clip,delta", [("none", None)] + [("adaptive", d) for d in DELTAS])
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "isolated", "switching"])
def test_torch_path_matches_float64_oracle_round_by_round(graph, clip, delta, attack):
    pr = LeastSquares(GRAPHS[graph], seed=1)
    byz = BYZ[graph] if attack else []
    conf = _conf(clip=clip, delta=delta) if clip == "adaptive" else _conf(clip="none")
    if attack:
        conf["byzantine"] = {"nodes": byz, "attack": attack, "scale": 2.0, "z": 1.5}
    opt = ClippedGossip(pr, "cpu", conf)
    theta = _np(opt.arena.theta)
    pub = theta.copy()
    for k in range(8):
        opt.run_rounds(1)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        if clip == "adaptive":                  # the radius choice must not hinge on rounding
            for i in range(W.shape[0]):
                # two ALIE attackers with the same honest neighbors publish the same row: an exact tie, which the
                # neighbor order decides on every path
                seen, nb = set(), []
                for j in co.neighbors(W, i):
                    if pub[j].tobytes() not in seen:
                        seen.add(pub[j].tobytes())
                        nb.append(j)
                d = np.array([np.linalg.norm(pub[j] - theta[i]) for j in nb])
                gap, pre = co.margins(d, np.array([W[i, j] for j in nb]), delta)
                assert gap > 1e-6 and pre > 1e-7, f"round {k} node {i}: test data too close to a tie"
        theta, pub, info = co.round_(theta, pub, W, pr.grad, 0.05, clip, delta or 0.0, _attack(byz, attack), 2.0, 1.5)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        np.testing.assert_allclose(_np(opt.pub), pub, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")


def test_link_drops_match_the_oracle_on_the_dropped_graphs():
    conf = _conf(alpha0=0.02, delta=0.2, outer_iterations=6,
                 byzantine={"nodes": [1], "attack": "alie", "z": 1.0})
    pr = _mnist_problem(conf)
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 6}
    pr._init_faults()
    opt = ClippedGossip(pr, "cpu", copy.deepcopy(conf))
    n = pr.layout.n
    graphs = set()
    for k in range(6):
        theta0, pub0 = _np(pr.arena.theta, n), _np(opt.pub, n)
        opt.run_rounds(1)
        W = pr.topology().W
        graphs.add(W.tobytes())
        mixed, _ = co.mix(theta0, pub0, W, "adaptive", 0.2)
        # the step is theta - alpha g: the mixed rows are recovered from theta + alpha g
        got = _np(pr.arena.theta, n) + opt.alph * _np(pr.arena.grad, n)
        np.testing.assert_allclose(got, mixed, rtol=0, atol=1e-5, err_msg=f"round {k}")
        hon = [j for j in co.neighbors(W, 1) if j != 1]
        if hon:
            x = pub0[hon]
            np.testing.assert_allclose(_np(opt.pub, n)[1], x.mean(0) - x.std(0), rtol=0, atol=1e-5)
    assert len(graphs) > 2


# --------------------------------------------------------------------------------------------- invariants ----
@pytest.mark.parametrize("delta", DELTAS)
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "switching"])
def test_clipping_invariants_every_round(graph, delta):
    pr = LeastSquares(GRAPHS[graph], seed=5)
    byz = BYZ[graph]
    attack = _attack(byz, "sign_flip")
    theta = 3.0 * np.random.default_rng(2).standard_normal((pr.N, 5))
    pub = theta.copy()
    for k in range(12):
        W = metropolis(GRAPHS[graph][k % len(GRAPHS[graph])])
        _, info = co.mix(theta, pub, W, "adaptive", delta)
        for i, (nb, d, f, tau) in enumerate(info):
            w = np.array([W[i, j] for j in nb])
            clipped = f < 1.0
            assert np.all(f <= 1.0) and np.all(f >= 0.0)
            assert np.all(f[~clipped] == 1.0)
            if tau > 0:
                assert np.all(f > 0.0)
            assert w[clipped].sum() <= delta + co.SLACK
            for e in np.nonzero(clipped)[0]:     # a clipped edge contributes at most W_ij tau
                assert np.linalg.norm(w[e] * f[e] * (pub[nb[e]] - theta[i])) <= w[e] * tau * (1 + 1e-12)
        theta, pub, _ = co.round_(theta, pub, W, pr.grad, 0.05, "adaptive", delta, attack, 3.0)


def test_delta_zero_is_dsgd_to_round_off():
    g = GRAPHS["random"]
    a = ClippedGossip(LeastSquares(g, seed=4), "cpu", _conf(delta=0.0))
    b = DSGD(LeastSquares(g, seed=4), "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.0, "outer_iterations": 50})
    for k in range(40):
        a.run_rounds(1)
        b.run_rounds(1)
    diff = (a.arena.theta - b.arena.theta).abs().max().item()
    print(f"\ndelta = 0 vs DSGD after 40 rounds: max difference {diff:.2e}")
    assert diff < 1e-13


@pytest.mark.parametrize("graph", ["switching", "random"])
def test_clip_none_without_attackers_is_dsgd_bitwise(graph):
    g = GRAPHS[graph]
    a = ClippedGossip(LeastSquares(g, seed=4), "cpu", _conf(clip="none", mu=0.3))
    b = DSGD(LeastSquares(g, seed=4), "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.3, "outer_iterations": 50})
    for k in range(20):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(a.arena.theta, b.arena.theta), f"round {k}"


# --------------------------------------------------------------------------------------------- robustness ----
class SharedMinimiser(LeastSquares):
    """Node i minimises 0.5 / m |A_i x - b_i|^2 with b_i = A_i x*: every node has the minimiser x*."""

    def __init__(self, graphs, seed=0):
        super().__init__(graphs, seed=seed)
        rng = np.random.default_rng(seed + 100)
        self.x_star = rng.standard_normal(self.A.shape[2])
        self.b = np.einsum("imn,n->im", self.A, self.x_star)
        self._b = torch.as_tensor(self.b, dtype=self._A.dtype)


@pytest.mark.parametrize("attack,scale,z", [("sign_flip", 10.0, 1.0), ("alie", 1.0, 10.0)])
def test_adaptive_clipping_keeps_the_honest_nodes_at_the_minimiser(attack, scale, z):
    """10-node complete graph, nodes 0 and 1 attack (weight 1/10 each), delta 0.2: without clipping the honest nodes
    end far from x* (or non-finite), with it they end at x*.  Oracle distances after 600 rounds (seed 0): sign flip
    (scale 10) 5.5e14 without clipping, 6.6e-9 with it; ALIE (z 10) 12.0 without, 6.2e-9 with."""
    R, err = 600, {}
    for clip in ("none", "adaptive"):
        pr = SharedMinimiser([nx.complete_graph(10)], seed=0)
        conf = _conf(clip=clip, delta=0.2, outer_iterations=R,
                     byzantine={"nodes": [0, 1], "attack": attack, "scale": scale, "z": z})
        opt = ClippedGossip(pr, "cpu", conf)
        opt.run_rounds(R)
        th = _np(opt.arena.theta)[2:]
        err[clip] = np.abs(th - pr.x_star).max() if np.isfinite(th).all() else np.inf
    print(f"\n{attack}: max |theta_honest - x*| " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert err["none"] > 1.0
    assert err["adaptive"] < 1e-6


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_refusals():
    assert ALGORITHMS["clipped_gossip"] is ClippedGossip
    base = {"alg_name": "clipped_gossip", "alpha0": 0.01, "clip": "none", "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["mu"] == 0.0 and c["update_graph"] is True and "byzantine" not in c
    for key in ("alpha0", "clip", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    with pytest.raises(ConfigError, match="clip"):
        validate_optimizer(dict(base, clip="median"))
    with pytest.raises(ConfigError, match="delta"):
        validate_optimizer(dict(base, clip="adaptive"))
    for dl in (1.0, -0.1, 1.5, "0.2", True):
        with pytest.raises(ConfigError, match="delta"):
            validate_optimizer(dict(base, clip="adaptive", delta=dl))
    validate_optimizer(dict(base, clip="adaptive", delta=0.0))
    byz = {"nodes": [0], "attack": "sign_flip"}
    validate_optimizer(dict(base, byzantine=byz))
    with pytest.raises(ConfigError, match=r"byzantine.*clipped_gossip only.*'dsgd'"):
        validate_optimizer({"alg_name": "dsgd", "alpha0": 0.1, "mu": 0.0, "outer_iterations": 3, "byzantine": byz})
    with pytest.raises(ConfigError, match="attack must be one of"):
        validate_optimizer(dict(base, byzantine=dict(byz, attack="label_flip")))
    with pytest.raises(ConfigError, match="duplicated"):
        validate_optimizer(dict(base, byzantine=dict(byz, nodes=[1, 1])))
    for key in ("scale", "z"):
        for v in (float("inf"), float("nan"), "1"):
            with pytest.raises(ConfigError, match=f"byzantine.{key} must be a finite number"):
                validate_optimizer(dict(base, byzantine=dict(byz, **{key: v})))
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(base, mixing_order="reference"))
    # node ids against the graph
    conf = _exp("cycle")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(base, byzantine=dict(byz, nodes=[4]))
    with pytest.raises(ConfigError, match="out of range"):
        validate_experiment(copy.deepcopy(conf), "mnist")
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(base, byzantine=dict(byz, nodes=[0, 1, 2, 3]))
    with pytest.raises(ConfigError, match="cover every node"):
        validate_experiment(copy.deepcopy(conf), "mnist")
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(base, byzantine=dict(byz, nodes=[3]))
    validate_experiment(copy.deepcopy(conf), "mnist")
    pr = LeastSquares(GRAPHS["cycle"])
    with pytest.raises(ValueError, match="attack must be one of"):
        ClippedGossip(pr, "cpu", _conf(byzantine={}))
    with pytest.raises(ValueError, match="out of range"):
        ClippedGossip(pr, "cpu", _conf(byzantine={"nodes": [6], "attack": "alie"}))
    with pytest.raises(ValueError, match="jacobi"):
        ClippedGossip(pr, "cpu", _conf(mixing_order="reference"))
    with pytest.raises(ValueError, match="undirected"):
        ClippedGossip(LeastSquares([nx.cycle_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())


def test_adaptive_clip_refuses_more_neighbors_than_the_mix_sorts():
    from nn_distributed_training_b200.ops.engine import CLIP_MAX_DEG, check_clip_capacity
    check_clip_capacity(CLIP_MAX_DEG)
    with pytest.raises(ValueError, match=f"at most {CLIP_MAX_DEG} neighbors per node.*a node with {CLIP_MAX_DEG + 1}"):
        check_clip_capacity(CLIP_MAX_DEG + 1)


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = {"alg_name": "clipped_gossip", "alpha0": 0.01,
                                                               "clip": "none", "outer_iterations": 3}
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'clipped_gossip'"):
        validate_experiment(conf, "mnist")


def test_byzantine_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_byzantine.yaml"), "mnist")
    assert conf["experiment"]["graph"]["type"] == "complete" and conf["experiment"]["graph"]["num_nodes"] == 10
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert ocs[0]["alg_name"] == "dsgd"
    arms = [(o["clip"], o["byzantine"]["attack"]) for o in ocs[1:]]
    assert arms == [("none", "sign_flip"), ("adaptive", "sign_flip"), ("none", "alie"), ("adaptive", "alie")]
    for o in ocs:
        assert o.get("complete_graph_mode") == "pointer"
        if o["alg_name"] == "clipped_gossip":
            assert len(o["byzantine"]["nodes"]) == 2 and (o["clip"] == "none" or o["delta"] == 0.2)


# ------------------------------------------------------------------------------------------------ runners ----
def test_mnist_runner_writes_byzantine_nodes_and_the_summary_is_honest_only(tmp_path, monkeypatch):
    from nn_distributed_training_b200.visualization.results import summarize_run
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_byzantine.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_byzantine"))
    assert len(out) == 1
    names = [pc["problem_name"] for pc in conf["problem_configs"].values()]
    for name in names:
        res = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        if name == names[0]:
            assert "byzantine_nodes" not in res
        else:
            assert res["byzantine_nodes"] == [0, 1]
        assert res["data_source"] == "synthetic"
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])
    s = summarize_run(out[0])
    res = torch.load(os.path.join(out[0], f"{names[-1]}_results.pt"), weights_only=False)
    acc = np.asarray(torch.as_tensor(res["top1_accuracy"][-1]))
    assert s[names[-1]]["final_top1_mean"] == pytest.approx(float(acc[2:].mean()))
    assert s[names[-1]]["final_top1_min"] == pytest.approx(float(acc[2:].min()))


def test_density_runner_runs_clipped_gossip(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="cg")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "clipped_gossip", "alpha0": 0.01, "clip": "adaptive", "delta": 0.2,
                              "outer_iterations": 4, "byzantine": {"nodes": [2], "attack": "sign_flip"}}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "cg_results.pt"), weights_only=False)
    assert res["byzantine_nodes"] == [2]
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def test_checkpoint_resume_with_an_alie_attacker_is_bit_exact(tmp_path):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, delta=0.2, outer_iterations=6, byzantine={"nodes": [1], "attack": "alie", "z": 1.0})
    full = _mnist_problem(conf)
    of = ClippedGossip(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = ClippedGossip(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    second = _mnist_problem(conf)
    o2 = ClippedGossip(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.pub, o1.pub)
    assert not torch.equal(o2.pub[1], second.arena.theta[1])      # the ALIE row is not the attacker's theta
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.pub, of.pub)
