"""K-GT and local DSGD on the PyTorch path (CPU): the float64 oracle round by round, the zero-sum correction, DSGT at
K = 1, DSGD bitwise at K = 1 without correction, exactness on heterogeneous least squares, configuration, the runners,
the draws per round and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import kgt_oracle as ko
from test_exact_diffusion import GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, DSGT, KGT, DiNNO
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
CORR = pytest.mark.parametrize("correction", [True, False], ids=["kgt", "local_dsgd"])


def _conf(**kw):
    return dict({"alg_name": "kgt", "alpha": 0.05, "local_steps": 2, "correction": True, "outer_iterations": 50}, **kw)


def _np(t, n=5):
    return t[:, :n].double().numpy().copy()


# ------------------------------------------------------------------------------------------------ oracle ----
@CORR
@pytest.mark.parametrize("K", [1, 2, 3, 5])
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "isolated", "switching"])
def test_torch_path_matches_float64_oracle_round_by_round(graph, K, correction):
    pr = LeastSquares(GRAPHS[graph], seed=1)
    opt = KGT(pr, "cpu", _conf(local_steps=K, correction=correction))
    theta = _np(opt.arena.theta)
    c = np.zeros_like(theta)
    y = np.zeros_like(theta)
    for k in range(8):
        opt.run_rounds(1)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        theta, c, y_new, _, _ = ko.round_(theta, c, y, W=W, grad_fn=pr.grad, alpha=0.05, K=K, correction=correction)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        if correction:
            y = y_new
            np.testing.assert_allclose(_np(opt.c), c, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
            np.testing.assert_allclose(_np(opt.y), y, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        else:
            assert opt.c is None and opt.y is None


def test_link_drops_match_the_oracle_on_the_dropped_graphs():
    """Link drops change the graph every round: the oracle walks the graph each round actually used."""
    conf = _conf(alpha=0.02, local_steps=3, outer_iterations=6)
    pr = _mnist_problem(conf)
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 6}
    pr._init_faults()
    opt = KGT(pr, "cpu", copy.deepcopy(conf))
    n = pr.layout.n
    c_sums, graphs = [], set()
    for k in range(6):
        before = (_np(pr.arena.theta, n), _np(opt.c, n), _np(opt.y, n))
        opt.run_rounds(1)
        W = pr.topology().W
        graphs.add(W.tobytes())
        x = ko.wmix(before[0], W)
        np.testing.assert_allclose(_np(opt.c, n), before[1] + ko.wmix(before[2], W) - before[2], rtol=0, atol=1e-6)
        c_sums.append(np.abs(_np(opt.c, n).sum(0)).max())
        assert np.abs(x - _np(pr.arena.theta, n)).max() > 0
    assert len(graphs) > 2
    assert max(c_sums) < 1e-5


# --------------------------------------------------------------------------------------------- invariants ----
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "switching"])
def test_correction_sums_to_zero_every_round(graph):
    pr = LeastSquares(GRAPHS[graph], seed=5)
    opt = KGT(pr, "cpu", _conf(local_steps=3))
    for k in range(20):
        opt.run_rounds(1)
        c = _np(opt.c)
        assert np.abs(c.sum(0)).max() <= 1e-13 * max(1.0, np.abs(c).max()), f"round {k}"


def test_one_local_step_is_dsgt():
    """K = 1: K-GT's tracker y = g + c is DSGT's (init_grads false), and K-GT's mixed row, theta + alpha y after the
    round, is DSGT's theta (DSGT's theta between rounds is the mixed row)."""
    alpha, R = 0.05, 300
    g = GRAPHS["random"]
    a = KGT(LeastSquares(g, seed=2), "cpu", _conf(alpha=alpha, local_steps=1, outer_iterations=R))
    b = DSGT(LeastSquares(g, seed=2), "cpu", {"alg_name": "dsgt", "alpha": alpha, "init_grads": False,
                                              "outer_iterations": R})
    diff, scale = [0.0, 0.0], [0.0, 0.0]
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        x = a.arena.theta + alpha * a.y
        for q, (got, want) in enumerate(((x, b.arena.theta), (a.y, b.y))):
            diff[q] = max(diff[q], (got - want).norm().item())
            scale[q] = max(scale[q], want.norm().item())
    # relative to the largest norm of the run: the trackers go to zero at the solution
    worst = max(d / s for d, s in zip(diff, scale))
    print(f"\nK-GT K=1 vs DSGT over {R} rounds: worst relative difference {worst:.2e}")
    assert worst < 1e-12


def test_local_dsgd_with_one_step_is_dsgd_bitwise():
    g = GRAPHS["switching"]
    a = KGT(LeastSquares(g, seed=4), "cpu", _conf(local_steps=1, correction=False))
    b = DSGD(LeastSquares(g, seed=4), "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.0, "outer_iterations": 50})
    for k in range(20):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(a.arena.theta, b.arena.theta), f"round {k}"


@pytest.mark.parametrize("K", [2, 4])
def test_kgt_reaches_the_global_least_squares_solution_where_local_dsgd_does_not(K):
    """Heterogeneous least squares, full deterministic gradients, cycle, constant step: K-GT converges to the minimiser
    of sum_i f_i; local DSGD (and DSGD) stop a measurable distance away."""
    rounds, alpha = 2000, 0.02
    err = {}
    for name, cls, conf in (("kgt", KGT, _conf(alpha=alpha, local_steps=K)),
                            ("local_dsgd", KGT, _conf(alpha=alpha, local_steps=K, correction=False)),
                            ("dsgd", DSGD, {"alg_name": "dsgd", "alpha0": alpha, "mu": 0.0})):
        pr = LeastSquares([nx.cycle_graph(8)], seed=3)
        opt = cls(pr, "cpu", dict(conf, outer_iterations=rounds))
        opt.run_rounds(rounds)
        err[name] = np.abs(_np(opt.arena.theta) - pr.solution()).max()
    print(f"\nK = {K}: max |theta - x*|: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert err["kgt"] < 1e-10
    assert err["local_dsgd"] > 1e-3 and err["dsgd"] > 1e-3


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["kgt"] is KGT
    base = {"alg_name": "kgt", "alpha": 0.01, "local_steps": 2, "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["correction"] is True and c["update_graph"] is True and c["profile"] is False
    for key in ("alpha", "local_steps", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    for ls in (0, -1, 2.0, 1.5, "2", True):
        with pytest.raises(ConfigError, match="local_steps"):
            validate_optimizer(dict(base, local_steps=ls))
    for alpha in (0.0, -0.1):
        with pytest.raises(ConfigError, match="alpha"):
            validate_optimizer(dict(base, alpha=alpha))
    with pytest.raises(ConfigError, match="correction"):
        validate_optimizer(dict(base, correction="yes"))
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(base, mixing_order="reference"))
    for key in ("update_graph", "consensus_backend", "checkpoint_every", "resume"):
        validate_optimizer(dict(base, **{key: True}))
    validate_optimizer(dict(base, correction=False, local_steps=1))
    pr = LeastSquares(GRAPHS["cycle"])
    with pytest.raises(ValueError, match="jacobi"):
        KGT(pr, "cpu", _conf(mixing_order="reference"))
    with pytest.raises(ValueError, match="local_steps"):
        KGT(pr, "cpu", _conf(local_steps=0))
    with pytest.raises(ValueError, match="alpha"):
        KGT(pr, "cpu", _conf(alpha=0.0))
    with pytest.raises(ValueError, match="undirected"):
        KGT(LeastSquares([nx.cycle_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = {"alg_name": "kgt", "alpha": 0.01, "local_steps": 2,
                                                               "outer_iterations": 3}
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'kgt'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")


def test_local_steps_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_local_steps.yaml"), "mnist")
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [(o["alg_name"], o.get("primal_iterations", o.get("local_steps")), o.get("correction")) for o in ocs] == [
        ("dinno", 2, None), ("dsgt", None, None), ("kgt", 2, False), ("kgt", 2, True)]
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    assert dict(conf["experiment"], name=None) == dict(paper["experiment"], name=None)
    assert conf["problem_configs"]["problem1"] == paper["problem_configs"]["problem1"]


# ------------------------------------------------------------------------------------------------ runners ----
def test_mnist_runner_on_the_local_steps_yaml(tmp_path, monkeypatch):
    """All four problems of the new YAML at a tiny size; K-GT with K = 2 draws as many batches as DiNNO with 2 primal
    steps."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_local_steps.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_local_steps"))
    assert len(out) == 1
    res = {}
    for name in ("dinno", "dsgt", "local_dsgd_k2", "kgt_k2"):
        res[name] = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert all(torch.isfinite(v).all() for v in res[name]["validation_loss"])
    fp = {k: [int(torch.as_tensor(v).sum()) for v in r["forward_pass_count"]] for k, r in res.items()}
    assert fp["kgt_k2"] == fp["dinno"] == fp["local_dsgd_k2"]
    assert fp["kgt_k2"][-1] > fp["dsgt"][-1]


def test_density_runner_runs_kgt(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="kgt")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "kgt", "alpha": 0.01, "local_steps": 3, "outer_iterations": 4}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "kgt_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


@pytest.mark.parametrize("K", [1, 3])
def test_draws_per_round_equal_local_steps(K):
    conf = _conf(alpha=0.02, local_steps=K, outer_iterations=4)
    a = _mnist_problem(conf)
    KGT(a, "cpu", copy.deepcopy(conf)).run_rounds(4)
    dconf = {"alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.0, "outer_iterations": 4, "primal_iterations": K,
             "primal_optimizer": "adam", "persistant_primal_opt": False, "primal_lr_start": 0.005,
             "primal_lr_finish": 0.005, "lr_decay_type": "constant"}
    b = _mnist_problem(dconf)
    DiNNO(b, "cpu", dconf).run_rounds(4)
    assert a.forward_cnt == b.forward_cnt
    assert a.forward_cnt == 4 * K * 32              # samples of one node: K batches of 32 per round


# ------------------------------------------------------------------------------------------------ resume ----
@CORR
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, correction):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha=0.02, local_steps=3, correction=correction, outer_iterations=6)
    full = _mnist_problem(conf)
    of = KGT(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = KGT(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = KGT(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3
    if correction:
        assert torch.equal(o2.c, o1.c) and torch.equal(o2.y, o1.y)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    if correction:
        assert torch.equal(o2.c, of.c) and torch.equal(o2.y, of.y)
    assert second.forward_cnt == full.forward_cnt
