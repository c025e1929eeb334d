"""SlowMo on the PyTorch path (CPU, float64): the outer update and one global and one gossip round against hand-computed
values, the NumPy oracle round by round over gossip and local SGD with and without base momentum, DSGD and DSGDm with
local momentum at a period past the run bit for bit, Gossip-PGA at slow_momentum 0 and slow_lr 1 within the oracle
bound, equal anchors, u and theta across nodes after every global round, the base momentum reset, every configuration
refusal and default, the runners, checkpoint/resume at and after a global round, and local SGD pulling nothing."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import slowmo_oracle as so
from hsgd_oracle import metropolis
from test_exact_diffusion import _mnist_problem, _synthetic
from test_gt_hsgd import GRAPHS, LSProblem, _np
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, DSGDm, GossipPGA, SlowMo
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
DROPS = {"link_drop_prob": 0.3, "seed": 5, "from_round": 2, "to_round": 12}
U64 = 2.0 ** -53


def _conf(**kw):
    return dict({"alg_name": "slowmo", "alpha0": 0.05, "mu": 0.5, "period": 3, "slow_momentum": 0.5,
                 "outer_iterations": 50}, **kw)


def _alphas(alpha0, mu, n):
    out, a = [], alpha0
    for _ in range(n):
        a = a * (1.0 - mu * a)
        out.append(a)
    return out


# ----------------------------------------------------------------------------------------- hand values ----
def test_outer_update_hand_computed():
    """u = 0.5 u + (a - xbar) / 0.5 and a -= (2 * 0.5) u, on values exact in binary; theta becomes a, m becomes 0."""
    theta = torch.tensor([[1.0, 2.0], [1.0, 2.0]], dtype=torch.float64)
    anchor = torch.tensor([[3.0, 0.0], [3.0, 0.0]], dtype=torch.float64)
    u = torch.tensor([[0.5, -1.0], [0.5, -1.0]], dtype=torch.float64)
    m = torch.ones(2, 2, dtype=torch.float64)
    ref.slowmo_outer_(theta, anchor, u, m, 0.5, 2.0, 0.5)
    assert u.tolist() == [[4.25, -4.5]] * 2
    assert anchor.tolist() == [[-1.25, 4.5]] * 2
    assert torch.equal(theta, anchor) and not m.any()


def test_one_global_and_one_gossip_round_hand_computed():
    """Two nodes joined by an edge (W = 1/2 everywhere), mu = 0, period 2: round 0 is a gossip round (anchor and u stay),
    round 1 global (gamma = alpha0)."""
    pr = LSProblem(nx.path_graph(2), batch=8, seed=1)
    a0, sm, sl = 0.05, 0.5, 1.5
    opt = SlowMo(pr, "cpu", _conf(alpha0=a0, mu=0.0, period=2, slow_momentum=sm, slow_lr=sl, outer_iterations=2))
    x0 = _np(pr.arena.theta)
    opt.run_rounds(1)
    x_mix = np.repeat(x0.mean(0, keepdims=True), 2, axis=0)              # W = [[1/2, 1/2], [1/2, 1/2]]
    x1 = x_mix - a0 * pr.batch_grad(x_mix, 0)
    np.testing.assert_allclose(_np(pr.arena.theta), x1, rtol=1e-14, atol=1e-14)
    assert np.array_equal(_np(opt.anchor), x0) and not opt.u.any()
    opt.run_rounds(1)
    xbar = x1.mean(0, keepdims=True)
    u = (x0 - xbar) / a0
    anchor = x0 - sl * a0 * u
    np.testing.assert_allclose(_np(opt.u), u, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(_np(opt.anchor), anchor, rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(_np(pr.arena.theta), anchor - a0 * pr.batch_grad(anchor, 1), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("base", [(0.0, False), (0.9, False), (0.9, True)], ids=["sgd", "momentum", "nesterov"])
@pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])
@pytest.mark.parametrize("drops", [False, True], ids=["static", "link_drops"])
@pytest.mark.parametrize("period", [1, 2, 3, 5])
@pytest.mark.parametrize("graph", ["cycle", "star", "random"])
def test_torch_path_matches_float64_oracle_round_by_round(graph, period, drops, gossip, base):
    R = 12
    bm, nest = base
    pr = LSProblem(GRAPHS[graph], batch=8, seed=1, faults=DROPS if drops else None)
    Ws = [metropolis(g) for g in pr.plan_graphs(R, 0, 1)]
    opt = SlowMo(pr, "cpu", _conf(period=period, gossip=gossip, base_momentum=bm, nesterov=nest, slow_lr=1.2,
                                  outer_iterations=R))
    want = so.run(_np(pr.arena.theta), Ws, _alphas(0.05, 0.5, R), 0.05, period, gossip, pr.batch_grad, R,
                  1.2, 0.5, bm, nest)
    for k, (theta, anchor, u) in enumerate(want):
        opt.run_rounds(1)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-10, atol=1e-10, err_msg=f"round {k}")
        np.testing.assert_allclose(_np(opt.anchor), anchor, rtol=1e-10, atol=1e-10, err_msg=f"round {k}")
        np.testing.assert_allclose(_np(opt.u), u, rtol=1e-9, atol=1e-9, err_msg=f"round {k}")
    assert pr.calls.tolist() == [R] * pr.N
    assert opt.alph == _alphas(0.05, 0.5, R)[-1]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_outer_update_within_the_oracle_bound(dtype):
    """``slowmo_outer_`` on random rows against the float64 oracle, |got - oracle| <= 16 err."""
    g = torch.Generator().manual_seed(0)
    rows = [torch.randn(3, 41, generator=g, dtype=torch.float64).to(dtype) for _ in range(3)]
    theta, anchor, u = (r.clone() for r in rows)
    gamma = float(torch.tensor(0.0371, dtype=dtype))
    ref.slowmo_outer_(theta, anchor, u, None, 0.0371, 1.3, 0.7)
    unit = U64 if dtype == torch.float64 else 2.0 ** -24
    un, eu, an, ea = so.slowmo_outer(*(r.double().numpy() for r in rows), gamma, 1.3, 0.7, unit)
    assert (np.abs(u.double().numpy() - un) <= 16 * eu).all()
    assert (np.abs(anchor.double().numpy() - an) <= 16 * ea).all()
    assert torch.equal(theta, anchor)


# ------------------------------------------------------------------------------------------ equivalences ----
@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_period_past_the_run_is_dsgd_bit_for_bit(model):
    R = 10
    sconf = _conf(period=R + 1, outer_iterations=R)
    dconf = {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": R}
    if model == "mnist":
        pa, pb = _mnist_problem(sconf), _mnist_problem(dconf)
    else:
        pa, pb = (LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS),
                  LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS))
    a, b = SlowMo(pa, "cpu", sconf), DSGD(pb, "cpu", dconf)
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"
        assert a.alph == b.alph
    assert pa.forward_cnt == pb.forward_cnt and (pa.calls == pb.calls).all()


@pytest.mark.parametrize("nesterov", [False, True], ids=["heavy_ball", "nesterov"])
@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_period_past_the_run_with_base_momentum_is_local_dsgdm_bit_for_bit(model, nesterov):
    R = 10
    sconf = _conf(period=R + 1, base_momentum=0.9, nesterov=nesterov, outer_iterations=R)
    dconf = {"alg_name": "dsgdm", "alpha0": 0.05, "mu": 0.5, "beta": 0.9, "momentum": "local", "nesterov": nesterov,
             "outer_iterations": R}
    if model == "mnist":
        pa, pb = _mnist_problem(sconf), _mnist_problem(dconf)
    else:
        pa, pb = (LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS),
                  LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS))
    a, b = SlowMo(pa, "cpu", sconf), DSGDm(pb, "cpu", dconf)
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"
        assert torch.equal(a.m, b.m), f"round {k}"


def _record_mixed(pr, out):
    """Record the row every node takes its gradient at (theta~) in ``out``."""
    orig = pr.compute_grads

    def probe():
        out.append(pr.arena.theta.clone())
        return orig()
    pr.compute_grads = probe


@pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])
@pytest.mark.parametrize("period", [1, 3])
def test_no_slow_momentum_and_unit_slow_lr_is_gossip_pga_within_the_oracle_bound(period, gossip):
    """Each round both optimizers start from SlowMo's rows.  A gossip round is Gossip-PGA's bit for bit; on a global round
    SlowMo's theta~ is Gossip-PGA's mean up to the outer update's rounding, a - gamma ((a - xbar) / gamma), which the
    oracle bounds (|diff| <= 16 err)."""
    R = 9
    pr, pq = LSProblem(GRAPHS["cycle"], batch=8, seed=3), LSProblem(GRAPHS["cycle"], batch=8, seed=3)
    conf = _conf(period=period, gossip=gossip, slow_momentum=0.0, slow_lr=1.0, outer_iterations=R)
    opt, pga = SlowMo(pr, "cpu", conf), GossipPGA(pq, "cpu", dict(conf, alg_name="gossip_pga"))
    mixed, mean = [], []
    _record_mixed(pr, mixed)
    _record_mixed(pq, mean)
    for k in range(R):
        pq.arena.theta.copy_(pr.arena.theta)
        anchor, u, gamma = _np(opt.anchor), _np(opt.u), opt.alph
        opt.run_rounds(1)
        pga.run_rounds(1)
        got, xbar = _np(mixed[-1]), _np(mean[-1])
        if not opt.is_global(k):
            assert np.array_equal(got, xbar) and torch.equal(pr.arena.theta, pq.arena.theta), f"round {k}"
            continue
        _, _, an, ea = so.slowmo_outer(xbar, anchor, u, gamma, 1.0, 0.0, U64)
        assert (np.abs(got - an) <= 16 * ea).all() and (np.abs(got - xbar) <= 16 * ea).all(), f"round {k}"


@pytest.mark.parametrize("base", [0.0, 0.9])
@pytest.mark.parametrize("gossip", [True, False], ids=["gossip", "local_sgd"])
@pytest.mark.parametrize("graph", ["cycle", "star", "random"])
def test_nodes_bitwise_equal_after_every_global_round(graph, gossip, base):
    """Identical initial rows (one model copied into every node): after each global round, before its step, anchors, u
    and theta~ are bitwise equal across nodes."""
    pr = LSProblem(GRAPHS[graph], batch=8, seed=2, faults=DROPS)
    pr.arena.theta.copy_(pr.arena.theta[0].expand_as(pr.arena.theta))
    opt = SlowMo(pr, "cpu", _conf(period=3, gossip=gossip, base_momentum=base, outer_iterations=12))
    mixed = []
    _record_mixed(pr, mixed)
    for k in range(12):
        opt.run_rounds(1)
        if opt.is_global(k):
            assert all(torch.equal(t[0].expand_as(t), t) for t in (mixed[-1], opt.anchor, opt.u)), f"round {k}"
            assert torch.equal(mixed[-1], opt.anchor)
    assert not torch.equal(pr.arena.theta[0].expand_as(pr.arena.theta), pr.arena.theta)


def test_base_momentum_reset_at_global_rounds():
    """After a global round m is that round's gradient alone (m <- 0 then m <- beta m + g); after a gossip round it is
    beta m + g of the previous m."""
    pr = LSProblem(GRAPHS["cycle"], batch=8, seed=4)
    opt = SlowMo(pr, "cpu", _conf(period=3, base_momentum=0.9, outer_iterations=9))
    for k in range(9):
        m_prev = opt.m.clone()
        opt.run_rounds(1)
        g = pr.arena.grad
        want = g if opt.is_global(k) or k == 0 else 0.9 * m_prev + g
        assert torch.equal(opt.m, want), f"round {k}"


def test_local_sgd_pulls_nothing():
    """gossip: false: only global rounds read other nodes' rows; gossip rounds touch neither the topology nor the
    gathered rows."""
    pr = LSProblem(GRAPHS["wheel"], batch=8, seed=4)
    opt = SlowMo(pr, "cpu", _conf(period=4, gossip=False, outer_iterations=12))
    calls = []
    gather, topology = pr.gather_rows, pr.topology
    pr.gather_rows = lambda t: (calls.append(("gather", opt.k)), gather(t))[1]
    pr.topology = lambda: (calls.append(("topology", opt.k)), topology())[1]
    opt.run_rounds(12)
    assert calls == [("gather", k) for k in (3, 7, 11)]


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "slowmo", "alpha0": 0.01, "period": 4, "slow_momentum": 0.5, "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["slowmo"] is SlowMo
    c = validate_optimizer(dict(BASE))
    assert (c["slow_lr"] == 1.0 and c["mu"] == 0.0 and c["gossip"] is True and c["base_momentum"] == 0.0
            and c["nesterov"] is False and c["update_graph"] is True and c["profile"] is False)
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, mu=0.1, period=1, gossip=False, slow_lr=2.0, slow_momentum=0.0, base_momentum=0.9,
                            nesterov=True, update_graph=False, profile=True))
    o = SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", dict(BASE))
    assert o.slow_lr == 1.0 and o.base_momentum == 0.0 and o.m is None and o.STATE == ("anchor", "u")
    assert o.gossip is True and o.nesterov is False and o.SCALARS == ("alph",)
    assert SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", dict(BASE, base_momentum=0.5)).STATE == ("anchor", "u", "m")


@pytest.mark.parametrize("key", ["alpha0", "period", "slow_momentum", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})
    if key != "outer_iterations":
        with pytest.raises(KeyError, match=key):
            SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", {k: v for k, v in _conf().items() if k != key})


@pytest.mark.parametrize("alpha0", [0.0, -0.1, float("inf"), float("nan"), "0.1", True])
def test_alpha0_must_be_finite_and_positive(alpha0):
    with pytest.raises(ConfigError, match="alpha0"):
        validate_optimizer(dict(BASE, alpha0=alpha0))
    if not isinstance(alpha0, (str, bool)):
        with pytest.raises(ValueError, match="alpha0"):
            SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(alpha0=alpha0))


@pytest.mark.parametrize("mu", [-0.1, float("inf"), "0.1", True])
def test_mu_must_be_finite_and_nonnegative(mu):
    with pytest.raises(ConfigError, match="mu"):
        validate_optimizer(dict(BASE, mu=mu))


def test_a_schedule_reaching_a_nonpositive_step_is_refused():
    """alpha_0 = 0.5 (1 - 2 * 0.5) = 0 and, with mu = 3, -0.25: gamma of round 1 would divide by it."""
    for mu, alpha in ((2.0, "0.0"), (3.0, "-0.25")):
        c = validate_optimizer(dict(BASE, alpha0=0.5, mu=mu, outer_iterations=3))
        with pytest.raises(ValueError, match=f"round 0 has alpha = {alpha}"):
            SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", c)
    SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", validate_optimizer(dict(BASE, alpha0=0.5, mu=1.0, outer_iterations=3)))


@pytest.mark.parametrize("period", [0, -2, 2.0, 1.5, "3", True, False])
def test_period_must_be_an_integer_of_at_least_one(period):
    with pytest.raises(ConfigError, match="period"):
        validate_optimizer(dict(BASE, period=period))
    with pytest.raises(ValueError, match="slowmo period"):
        SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(period=period))


@pytest.mark.parametrize("key", ["slow_momentum", "base_momentum"])
@pytest.mark.parametrize("v", [-0.1, 1.0, 1.5, "0.5", True, None])
def test_momenta_must_be_in_unit_interval(key, v):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer(dict(BASE, **{key: v}))
    with pytest.raises(ValueError, match=key):
        SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(**{key: v}))


@pytest.mark.parametrize("v", [0.0, -1.0, float("inf"), float("nan"), "1", True])
def test_slow_lr_must_be_finite_and_positive(v):
    with pytest.raises(ConfigError, match="slow_lr"):
        validate_optimizer(dict(BASE, slow_lr=v))
    with pytest.raises(ValueError, match="slow_lr"):
        SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(slow_lr=v))


@pytest.mark.parametrize("key", ["gossip", "nesterov"])
@pytest.mark.parametrize("v", [1, 0, "true", None])
def test_switches_must_be_bools(key, v):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer(dict(BASE, **{key: v}))
    with pytest.raises(ValueError, match=key):
        SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(**{key: v}))


@pytest.mark.parametrize("key", ["beta", "momentum", "alpha", "local_steps", "gossip_steps"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"slowmo takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="slowmo runs the synchronous"):
        SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="slowmo does not model Byzantine"):
        SlowMo(LSProblem(GRAPHS["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'slowmo'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="slowmo needs an undirected"):
        SlowMo(LSProblem(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())


def test_changing_graphs_and_link_drops_are_accepted():
    pr = LSProblem(GRAPHS["cycle"], faults=dict(DROPS, from_round=0, to_round=6))
    assert len({tuple(sorted(g.edges())) for g in pr.plan_graphs(6, 0, 1)}) > 1
    SlowMo(pr, "cpu", _conf(outer_iterations=6)).run_rounds(6)
    assert np.isfinite(pr.arena.theta.numpy()).all()


# ------------------------------------------------------------------------------------------------ runners ----
ARMS = [("dsgd", None, None, None, None), ("gossip_pga", 4, True, None, None), ("gossip_pga", 4, False, None, None),
        ("slowmo", 4, True, 0.5, 0.0), ("slowmo", 4, False, 0.5, 0.0), ("slowmo", 4, True, 0.5, 0.9)]
NAMES = ["dsgd", "gossip_pga_p4", "local_sgd_p4", "slowmo_p4", "slowmo_local_p4", "slowmo_p4_bm09"]


def test_slowmo_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_slowmo.yaml"), "mnist")
    pcs = list(conf["problem_configs"].values())
    ocs = [p["optimizer_config"] for p in pcs]
    assert [(o["alg_name"], o.get("period"), o.get("gossip"), o.get("slow_momentum"), o.get("base_momentum"))
            for o in ocs] == ARMS
    assert [p["problem_name"] for p in pcs] == NAMES
    assert all(p["train_batch_size"] == 64 for p in pcs)
    assert all(o["alpha0"] == 0.005 and o["mu"] == 0.001 and o["outer_iterations"] == 2000 for o in ocs)
    e = conf["experiment"]
    assert e["graph"]["type"] == "cycle" and e["graph"]["num_nodes"] == 10 and e["data_split_type"] == "hetero"


def test_mnist_runner_on_the_slowmo_yaml(tmp_path, monkeypatch):
    """The six problems of the YAML at a tiny size, written and read back with visualization.results; every arm draws
    one batch per round."""
    from nn_distributed_training_b200.visualization.results import load_results
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_slowmo.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_slowmo"))
    assert len(out) == 1
    fp = {}
    for name in NAMES:
        res = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])
        fp[name] = [int(torch.as_tensor(v).sum()) for v in res["forward_pass_count"]]
    assert len({tuple(v) for v in fp.values()}) == 1
    assert set(NAMES) <= set(load_results(out[0]))


def test_density_runner_runs_slowmo(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="slowmo")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "slowmo", "alpha0": 0.01, "period": 2, "slow_momentum": 0.5,
                              "outer_iterations": 4}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "slowmo_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("base", [0.0, 0.9], ids=["sgd", "momentum"])
@pytest.mark.parametrize("stop", [5, 6], ids=["at_global_round", "after_global_round"])
def test_checkpoint_resume_is_bit_exact(tmp_path, stop, base):
    """period 3: round 5 is global, so stopping after 5 rounds resumes at a global round and after 6 at the round after
    it; anchor, u and m resume with theta."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, period=3, base_momentum=base, outer_iterations=9)
    assert SlowMo(_mnist_problem(conf), "cpu", copy.deepcopy(conf)).is_global(5)
    full = _mnist_problem(conf)
    of = SlowMo(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = SlowMo(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=stop, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = stop                   # "crash" after round `stop`
    o1.train()
    assert o1.k == stop
    second = _mnist_problem(conf)
    o2 = SlowMo(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=stop, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == stop and o2.alph == o1.alph
    assert torch.equal(o2.anchor, o1.anchor) and torch.equal(o2.u, o1.u) and o2.u.any()
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.anchor, of.anchor) and torch.equal(o2.u, of.u)
    if base:
        assert torch.equal(o2.m, of.m)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt
