"""BEER on the PyTorch path (CPU): a float64 oracle round by round, the invariants that show every code is applied once
and the tracker tracks, DSGT equivalence, exactness on heterogeneous least squares where CHOCO-SGD and DSGD stay biased,
configuration, the MNIST runner and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import beer_oracle as bo
import choco_oracle as cho
from test_exact_diffusion import GRAPHS, LeastSquares, metropolis
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, BEER, DSGD, DSGT, ChocoSGD
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
STATIC = {k: v for k, v in GRAPHS.items() if k != "switching"}
COMPRESSORS = ["none", "int8", "sign"]


def _conf(comp, **kw):
    return dict({"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "compressor": comp, "outer_iterations": 50}, **kw)


def _np(t):
    return t.detach().double().cpu().numpy().copy()


def _nbrs(W):
    return [[j for j in range(W.shape[0]) if j != i and W[i, j] != 0] for i in range(W.shape[0])]


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("graph", sorted(STATIC))
def test_torch_path_matches_float64_oracle_round_by_round(graph, comp):
    """Each round against the oracle: the mix from the pending codes, then the tracker update with the round's gradient.
    The codes are the encoder's (its bytes are tested in test_choco.py), so the oracle takes h' = h + dec(qh) and
    g' = g + dec(qg) from the published rows and continues from the optimizer's state."""
    pr = LeastSquares(STATIC[graph], seed=1)
    opt = BEER(pr, "cpu", _conf(comp))
    W = metropolis(STATIC[graph][0])
    nbrs = _nbrs(W)
    n_pad, live = opt.arena.n_pad, opt.live.numpy()
    u = 2.0 ** -53
    dec = lambda code: np.stack([cho.decode(code[i], comp, n_pad, np.float64, live)[0] for i in range(pr.N)])
    for k in range(8):
        st = {n: _np(getattr(opt, n)) for n in ("h", "s_h", "v", "g", "s_g", "m_old")}
        theta = _np(opt.arena.theta)
        dh, dg = dec(opt.code_h.numpy()), dec(opt.code_g.numpy())
        opt.run_rounds(1)
        th, sh, sg, e_th, e_sh, e_sg = bo.mix(theta, st["h"], st["s_h"], st["v"], st["s_g"], dh, dg, nbrs, W, 0.5,
                                              0.05, u, 0.0)
        grad = np.zeros_like(th)
        grad[:, :5] = np.stack([pr.grad(i, th[i, :5]) for i in range(pr.N)])
        v, e_v = bo.step_tracker(st["v"], st["g"], sg, st["m_old"], grad, 0.0, 0.5, u)
        for name, got, want, err in (("theta", _np(opt.arena.theta), th, e_th), ("s_h", _np(opt.s_h), sh, e_sh),
                                     ("s_g", _np(opt.s_g), sg, e_sg), ("v", _np(opt.v), v, e_v)):
            np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-12, err_msg=f"round {k} {name}")
        np.testing.assert_allclose(_np(opt.m_old), grad, rtol=1e-11, atol=1e-12, err_msg=f"round {k} m_old")
        # the estimates take exactly the decoded codes published this round
        assert np.array_equal(_np(opt.h), st["h"] + dec(opt.code_h.numpy())), f"round {k} h"
        assert np.array_equal(_np(opt.g), st["g"] + dec(opt.code_g.numpy())), f"round {k} g"


# ---------------------------------------------------------------------------------------- invariants ----
@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("graph", ["random", "wheel", "isolated"])
def test_invariants_hold_every_round(graph, comp):
    """Every round: s_h + W dec(qh pending) == W h and s_g + W dec(qg pending) == W g (every code applied once);
    sum_i v_i == sum_i m_old_i (the tracker tracks the sum of the latest gradients); sum_i theta_i moves by
    -alpha sum_i v_i (W is doubly stochastic: the gossip term sums to zero)."""
    g = STATIC[graph][0]
    pr = LeastSquares([g], seed=4)
    opt = BEER(pr, "cpu", _conf(comp, outer_iterations=100))
    W = torch.as_tensor(metropolis(g))
    n_pad = opt.arena.n_pad
    worst = dict(s=0.0, v=0.0, theta=0.0)
    for _ in range(100):
        sum0, vsum0 = opt.arena.theta.sum(0).clone(), opt.v.sum(0).clone()
        opt.run_rounds(1)
        for s, est, code in ((opt.s_h, opt.h, opt.code_h), (opt.s_g, opt.g, opt.code_g)):
            want = W @ est
            got = s + W @ ref.choco_decode(code, comp, n_pad, torch.float64, opt.live)
            worst["s"] = max(worst["s"], (got - want).abs().max().item() / max(est.abs().max().item(), 1e-300))
        scale = max(opt.m_old.abs().max().item(), 1e-300)
        worst["v"] = max(worst["v"], (opt.v.sum(0) - opt.m_old.sum(0)).abs().max().item() / scale)
        moved = opt.arena.theta.sum(0) - sum0
        worst["theta"] = max(worst["theta"], (moved + 0.05 * vsum0).abs().max().item()
                             / max(opt.arena.theta.abs().max().item(), 1e-300))
    print(f"\n{graph} {comp}: |s - W est| {worst['s']:.1e}, |sum v - sum m_old| {worst['v']:.1e}, "
          f"|sum theta step + alpha sum v| {worst['theta']:.1e}")
    assert worst["s"] < 1e-13 and worst["v"] < 1e-12 and worst["theta"] < 1e-12


@pytest.mark.parametrize("graph", ["cycle", "wheel", "isolated"])
def test_none_with_gamma_one_equals_dsgt_own_tracker(graph):
    """compressor none, gamma 1, from a common starting row: BEER's iterates are DSGT's with own_tracker_step and no
    initial gradient draw (theta <- W theta - alpha y, y <- W y + g - g_old), up to rounding."""
    pr = LeastSquares(STATIC[graph], seed=5)
    b = BEER(pr, "cpu", _conf("none", gamma=1.0, outer_iterations=300))
    b.arena.theta[:] = b.arena.theta[0].clone()
    b.run_rounds(300)
    pr2 = LeastSquares(STATIC[graph], seed=5)
    d = DSGT(pr2, "cpu", {"alg_name": "dsgt", "alpha": 0.05, "init_grads": False, "own_tracker_step": True,
                          "outer_iterations": 300, "update_graph": False})
    d.arena.theta[:] = d.arena.theta[0].clone()
    d.run_rounds(300)
    r = np.abs(_np(b.arena.theta) - _np(d.arena.theta)).max() / np.abs(_np(d.arena.theta)).max()
    # the trackers shrink towards the mean gradient, 0 at the solution: measured against the gradients' scale
    rv = np.abs(_np(b.v) - _np(d.y)).max() / np.abs(_np(d.g)).max()
    print(f"\nbeer none gamma=1 vs dsgt own tracker ({graph}): theta {r:.2e}, tracker {rv:.2e}")
    assert r < 1e-12 and rv < 1e-12


# --------------------------------------------------------------------------------------------- exactness ----
def _rel_to_solution(opt, pr):
    x = pr.solution()
    th = _np(opt.arena.theta)[:, :len(x)]
    return np.abs(th - x).max() / np.abs(x).max()


@pytest.mark.parametrize("comp", ["int8", "sign"])
def test_compressed_beer_is_exact_on_heterogeneous_least_squares(comp):
    """Full gradients, heterogeneous local minimisers, a 10-node cycle: BEER with int8 or sign codes reaches the global
    least-squares solution at every node; CHOCO-SGD with the same codes and DSGD, at the same constant step, keep the
    heterogeneity bias."""
    g = [nx.cycle_graph(10)]
    R, alpha, gamma = 3000, 0.05, 0.5
    pr = LeastSquares(g, n=20, m=40, seed=6)
    b = BEER(pr, "cpu", _conf(comp, alpha=alpha, gamma=gamma, outer_iterations=R))
    b.run_rounds(R)
    rb = _rel_to_solution(b, pr)
    pc = LeastSquares(g, n=20, m=40, seed=6)
    c = ChocoSGD(pc, "cpu", {"alg_name": "choco_sgd", "alpha0": alpha, "mu": 0.0, "gamma": gamma, "compressor": comp,
                             "outer_iterations": R})
    c.run_rounds(R)
    rc = _rel_to_solution(c, pc)
    pd = LeastSquares(g, n=20, m=40, seed=6)
    d = DSGD(pd, "cpu", {"alg_name": "dsgd", "alpha0": alpha, "mu": 0.0, "outer_iterations": R})
    d.run_rounds(R)
    rd = _rel_to_solution(d, pd)
    print(f"\n{comp}, {R} rounds: max relative distance to the solution: BEER {rb:.1e}, CHOCO {rc:.1e}, DSGD {rd:.1e}")
    assert rb < 1e-9
    assert rc > 1e-2 and rd > 1e-2


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["beer"] is BEER
    base = {"alg_name": "beer", "alpha": 0.01, "gamma": 0.5, "compressor": "int8", "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["update_graph"] is False and c["profile"] is False
    for key in ("alpha", "gamma", "compressor", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    for bad in ({"gamma": 0.0}, {"gamma": 1.5}, {"compressor": "top_k"}, {"mixing_order": "reference"},
                {"update_graph": True}):
        with pytest.raises(ConfigError, match=next(iter(bad))):
            validate_optimizer(dict(base, **bad))
    validate_optimizer(dict(base, gamma=1.0, update_graph=False))
    pr = LeastSquares(GRAPHS["cycle"])
    for bad, msg in (({"mixing_order": "reference"}, "jacobi"), ({"update_graph": True}, "fixed graph"),
                     ({"gamma": 0.0}, "gamma"), ({"gamma": 1.01}, "gamma"), ({"compressor": "fp16"}, "compressor")):
        with pytest.raises(ValueError, match=msg):
            BEER(pr, "cpu", _conf("int8", **bad))


def test_a_directed_graph_is_refused():
    with open(os.path.join(EXP, "dist_mnist_beer.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"]["graph"] = {"num_nodes": 10, "type": "directed_cycle"}
    conf["problem_configs"] = {"p": conf["problem_configs"]["problem3"]}
    with pytest.raises(ConfigError, match="directed"):
        validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        BEER(LeastSquares([nx.DiGraph(nx.cycle_graph(5))]), "cpu", _conf("int8"))


def test_a_changing_graph_is_refused():
    pr = _mnist_problem(_conf("int8"))
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 1}
    with pytest.raises(ValueError, match="fault_injection"):
        BEER(pr, "cpu", _conf("int8"))
    # a graph sequence that changes during the run (a moving plan), on the PyTorch path
    opt = BEER(LeastSquares(GRAPHS["switching"]), "cpu", _conf("int8"))
    opt.pr.plan_graphs = lambda oits, k0, dpr, init=0, refresh=True: [nx.cycle_graph(6), nx.path_graph(6)] * oits
    with pytest.raises(ValueError, match="beer needs a fixed graph"):
        opt.run_rounds(1)


def test_beer_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_beer.yaml"), "mnist")
    opts = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [o["alg_name"] for o in opts] == ["dsgt", "choco_sgd", "beer", "beer"]
    assert [o.get("compressor") for o in opts[1:]] == ["int8", "int8", "sign"]
    assert opts[0]["alpha"] == opts[2]["alpha"] == opts[3]["alpha"] == 0.005 and opts[0]["init_grads"]
    assert conf["experiment"]["data_split_type"] == "hetero"
    choco = load_experiment(os.path.join(EXP, "dist_mnist_choco.yaml"), "mnist")
    for key in ("graph", "model", "data_split_type"):
        assert conf["experiment"][key] == choco["experiment"][key]
    for p in conf["problem_configs"].values():
        assert p["train_batch_size"] == 64 and p["optimizer_config"]["outer_iterations"] == 2000


# ------------------------------------------------------------------------------------------------ runner ----
def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch):
    from test_exact_diffusion import _synthetic
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="beer")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "beer", "alpha": 0.01, "gamma": 0.5, "compressor": "sign",
                              "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    assert {"graph.gpickle", "beer_results.pt"} <= set(os.listdir(outs[0]))
    res = torch.load(os.path.join(outs[0], "beer_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"}
    assert len(res["validation_loss"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def _mnist_problem(conf, N=4, M=100):
    from test_exact_diffusion import _mnist_problem as mk
    return mk(conf, N=N, M=M)


@pytest.mark.parametrize("comp", COMPRESSORS)
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, comp):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(comp, alpha=0.02, outer_iterations=6)
    full = _mnist_problem(conf)
    of = BEER(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = BEER(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = BEER(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and all(torch.equal(getattr(o2, n), getattr(o1, n)) for n in BEER.STATE)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for n in BEER.STATE:
        assert torch.equal(getattr(o2, n), getattr(of, n)), n
    assert second.forward_cnt == full.forward_cnt
