"""DSGD with momentum on the PyTorch path (CPU): the float64 oracle round by round, DSGD at beta = 0, the mean
invariants of both momentum modes, the fixed points that tell the modes apart, configuration, the MNIST runner and
checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import dsgdm_oracle as mo
from test_exact_diffusion import GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, DSGDm
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
VARIANTS = [("local", False), ("local", True), ("quasi_global", False), ("quasi_global", True)]
VARIANT = pytest.mark.parametrize("momentum,nesterov", VARIANTS, ids=["local", "local-nest", "qg", "qg-nest"])
BETA = 0.8


def _conf(**kw):
    return dict({"alg_name": "dsgdm", "alpha0": 0.05, "mu": 0.0, "beta": BETA, "momentum": "local",
                 "outer_iterations": 50}, **kw)


def _theta(opt):
    return opt.arena.theta[:, :opt.pr.layout.n].double().numpy().copy()


def _row(t, n=5):
    return t[:, :n].double().numpy().copy()


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("mu", [0.0, 0.7])
@VARIANT
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph, momentum, nesterov, mu):
    pr = LeastSquares(GRAPHS[graph], seed=1)
    opt = DSGDm(pr, "cpu", _conf(mu=mu, momentum=momentum, nesterov=nesterov))
    qg = momentum == "quasi_global"
    theta, m, xp = _theta(opt), None, None
    alpha = 0.05
    for k in range(8):
        opt.run_rounds(1)
        alpha_prev, alpha = alpha, alpha * (1.0 - mu * alpha)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        theta, m, xp, _ = mo.round_(theta, m, xp, k=k, W=W, grad_fn=pr.grad, alpha=alpha, alpha_prev=alpha_prev,
                                    beta=BETA, quasi_global=qg, nesterov=nesterov)
        np.testing.assert_allclose(_theta(opt), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        np.testing.assert_allclose(_row(opt.m), m, rtol=1e-12, atol=1e-11, err_msg=f"round {k}")
        if qg:
            np.testing.assert_allclose(_row(opt.x_prev), xp, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        else:
            assert opt.x_prev is None
    assert opt.alph == pytest.approx(alpha, rel=1e-15)


@VARIANT
def test_beta_zero_is_dsgd_bitwise(momentum, nesterov):
    g = GRAPHS["switching"]
    a = DSGDm(LeastSquares(g, seed=4), "cpu", _conf(mu=0.7, beta=0.0, momentum=momentum, nesterov=nesterov))
    b = DSGD(LeastSquares(g, seed=4), "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.7, "outer_iterations": 50})
    for k in range(10):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(a.arena.theta, b.arena.theta), f"round {k}"
    assert a.alph == b.alph


@VARIANT
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "switching"])
def test_mean_invariants_on_doubly_stochastic_graphs(graph, momentum, nesterov):
    """local: mean m' = beta mean m + mean g.  quasi-global: the mean displacement d of round k is the mean step
    direction of round k - 1 (W doubly stochastic keeps the mean through the mix)."""
    pr = LeastSquares(GRAPHS[graph], seed=5)
    mu = 0.7
    opt = DSGDm(pr, "cpu", _conf(mu=mu, momentum=momentum, nesterov=nesterov))
    n = pr.A.shape[2]
    alphas = opt.alpha_table()
    prev_dir = m_old = xp_old = None
    for k in range(12):
        if k > 0:
            m_old = _row(opt.m, n)
            xp_old = None if opt.x_prev is None else _row(opt.x_prev, n)
        opt.run_rounds(1)
        g = _row(opt.arena.grad, n)
        m = _row(opt.m, n)
        if momentum == "local":
            want = g.mean(0) if k == 0 else BETA * m_old.mean(0) + g.mean(0)
            np.testing.assert_allclose(m.mean(0), want, rtol=0, atol=1e-13 * max(1.0, np.abs(m).max()))
            mom = m
        else:
            if k > 0:
                d = (xp_old - _row(opt.x_prev, n)) / alphas[k - 1]
                np.testing.assert_allclose(d.mean(0), prev_dir.mean(0), rtol=0,
                                           atol=1e-11 * max(1.0, np.abs(prev_dir).max()), err_msg=f"round {k}")
            mom = BETA * m + g
        prev_dir = g + BETA * mom if nesterov else mom


def _run_to_fixed_point(cls, conf, rounds):
    pr = LeastSquares([nx.cycle_graph(8)], seed=3)
    opt = cls(pr, "cpu", dict(conf, outer_iterations=rounds))
    opt.run_rounds(rounds)
    return _theta(opt)


@VARIANT
def test_fixed_points_tell_the_modes_apart(momentum, nesterov):
    """Heterogeneous least squares, full gradients, cycle, constant step.  Local momentum ends at DSGD's fixed point at
    step alpha / (1 - beta) (m = g / (1 - beta) there); quasi-global at DSGD's at alpha, or alpha (1 + beta) with
    Nesterov (the displacement d, and so mhat, vanish: m = g)."""
    alpha, beta, rounds = 0.02, 0.5, 4000
    got = _run_to_fixed_point(DSGDm, _conf(alpha0=alpha, beta=beta, momentum=momentum, nesterov=nesterov), rounds)
    if momentum == "local":
        eff, other = alpha / (1.0 - beta), alpha * (1.0 + beta) if nesterov else alpha
    else:
        eff, other = (alpha * (1.0 + beta) if nesterov else alpha), alpha / (1.0 - beta)
    dsgd = {"alg_name": "dsgd", "mu": 0.0}
    want = _run_to_fixed_point(DSGD, dict(dsgd, alpha0=eff), 2 * rounds)
    wrong = _run_to_fixed_point(DSGD, dict(dsgd, alpha0=other), 2 * rounds)
    err = np.abs(got - want).max()
    print(f"\n{momentum} nesterov={nesterov}: |theta - DSGD(alpha={eff:.4g})|_max {err:.2e}, "
          f"to DSGD(alpha={other:.4g}) {np.abs(got - wrong).max():.2e}")
    assert err < 1e-10 * max(1.0, np.abs(want).max())
    assert np.abs(got - wrong).max() > 1e6 * err


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["dsgdm"] is DSGDm
    base = {"alg_name": "dsgdm", "alpha0": 0.01, "beta": 0.9, "momentum": "quasi_global", "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["mu"] == 0.0 and c["nesterov"] is False and c["update_graph"] is True and c["profile"] is False
    for key in ("alpha0", "beta", "momentum", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    for beta in (-0.1, 1.0, 1.5):
        with pytest.raises(ConfigError, match="beta"):
            validate_optimizer(dict(base, beta=beta))
    validate_optimizer(dict(base, beta=0.0))
    with pytest.raises(ConfigError, match="momentum"):
        validate_optimizer(dict(base, momentum="global"))
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(base, mixing_order="reference"))
    for key in ("update_graph", "consensus_backend", "checkpoint_every", "resume"):
        validate_optimizer(dict(base, **{key: True}))
    with pytest.raises(ValueError, match="jacobi"):
        DSGDm(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))
    with pytest.raises(ValueError, match="beta"):
        DSGDm(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(beta=1.0))
    with pytest.raises(ValueError, match="momentum"):
        DSGDm(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(momentum="global"))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = {"alg_name": "dsgdm", "alpha0": 0.01, "beta": 0.9,
                                                               "momentum": "local", "outer_iterations": 3}
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'dsgdm'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")


def test_quasi_global_refuses_a_schedule_reaching_zero():
    """alpha_0 = alpha0 (1 - mu alpha0) is 0 for alpha0 = 2, mu = 0.5 and negative for alpha0 = 1, mu = 2 (and every
    later entry then stays <= 0).  Local momentum does not divide by it."""
    pr = LeastSquares(GRAPHS["cycle"])
    with pytest.raises(ValueError, match=r"round 0 has alpha = 0\.0"):
        DSGDm(pr, "cpu", _conf(alpha0=2.0, mu=0.5, momentum="quasi_global"))
    with pytest.raises(ValueError, match=r"round 0 has alpha = -1\.0"):
        DSGDm(pr, "cpu", _conf(alpha0=1.0, mu=2.0, momentum="quasi_global"))
    DSGDm(pr, "cpu", _conf(alpha0=2.0, mu=0.5, momentum="local"))


def test_momentum_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_momentum.yaml"), "mnist")
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [(o["alg_name"], o.get("momentum"), o.get("nesterov")) for o in ocs] == [
        ("dsgd", None, None), ("dsgdm", "local", True), ("dsgdm", "quasi_global", True)]
    hetero = load_experiment(os.path.join(EXP, "dist_mnist_hetero_ed.yaml"), "mnist")
    assert dict(conf["experiment"], name=None) == dict(hetero["experiment"], name=None)


# ------------------------------------------------------------------------------------------------ runner ----
def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="dsgdm")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "dsgdm", "alpha0": 0.01, "beta": 0.9, "momentum": "quasi_global",
                              "nesterov": True, "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    files = set(os.listdir(outs[0]))
    assert {"graph.gpickle", "dsgdm_results.pt"} <= files
    res = torch.load(os.path.join(outs[0], "dsgdm_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"}
    assert len(res["validation_loss"]) == 3          # rounds 0, 2 and 4 (the last)
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("momentum", ["local", "quasi_global"])
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, momentum):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, beta=0.9, momentum=momentum, nesterov=True, outer_iterations=6)
    full = _mnist_problem(conf)
    of = DSGDm(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = DSGDm(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = DSGDm(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.m, o1.m)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.m, of.m)
    if momentum == "quasi_global":
        assert torch.equal(o2.x_prev, of.x_prev)
    assert o2.alph == of.alph
    assert second.forward_cnt == full.forward_cnt
