"""DeTAG on the PyTorch path (CPU, float64): the NumPy oracle round by round, the mixing rate and the Chebyshev weights,
the contraction of one multi-step gossip, the tracking invariant, DSGT at K = 1, exactness on heterogeneous least
squares, every configuration refusal, the runners and checkpoint/resume."""
import copy
import glob
import math
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import detag_oracle as do
from test_exact_diffusion import GRAPHS as ED_GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, DSGT, DeTAG
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
ACC = pytest.mark.parametrize("accelerate", [True, False], ids=["chebyshev", "plain"])
GRAPHS = {
    "cycle": nx.cycle_graph(8),
    "path": nx.path_graph(6),
    "star": nx.star_graph(6),
    "wheel": nx.wheel_graph(7),
    "random": ED_GRAPHS["random"][0],
    "complete": nx.complete_graph(6),
    "binary_tree": nx.balanced_tree(2, 3),
}


def _conf(**kw):
    return dict({"alg_name": "detag", "alpha": 0.05, "gossip_steps": 2, "accelerate": True, "outer_iterations": 50}, **kw)


def _np(t, n=5):
    return t[:, :n].double().numpy().copy()


def _cycle_lambda(N):
    return 1.0 / 3.0 + (2.0 / 3.0) * math.cos(2.0 * math.pi / N)


# ------------------------------------------------------------------------------------------------ oracle ----
@ACC
@pytest.mark.parametrize("K", [1, 2, 3, 5])
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph, K, accelerate):
    pr = LeastSquares([GRAPHS[graph]], seed=1)
    opt = DeTAG(pr, "cpu", _conf(gossip_steps=K, accelerate=accelerate))
    W = metropolis(GRAPHS[graph])
    omega = do.weights(do.lam(W), K, accelerate)
    np.testing.assert_allclose(opt.omega, omega, rtol=1e-12, atol=0)
    z = _np(opt.arena.theta)
    y = np.zeros_like(z)
    g_old = np.zeros_like(z)
    for k in range(8):
        opt.run_rounds(1)
        theta, y, g_old, z = do.round_(z, y, g_old, W=W, grad_fn=pr.grad, alpha=0.05, omega=omega)
        for name, got, want in (("theta", opt.arena.theta, theta), ("y", opt.y, y), ("g_old", opt.g_old, g_old),
                                ("z", opt.z, z)):
            np.testing.assert_allclose(_np(got), want, rtol=1e-11, atol=1e-11, err_msg=f"round {k}: {name}")


@pytest.mark.parametrize("N", [4, 5, 10, 32])
def test_cycle_lambda_and_weights_match_the_closed_form(N):
    pr = LeastSquares([nx.cycle_graph(N)], seed=0)
    opt = DeTAG(pr, "cpu", _conf(gossip_steps=8))
    lam = _cycle_lambda(N)
    assert opt.lam == pytest.approx(lam, rel=1e-13, abs=1e-15)
    np.testing.assert_allclose(opt.omega, do.weights(lam, 8), rtol=1e-12, atol=0)
    assert opt.omega[0] == 1.0 and opt.omega[1] == pytest.approx(2.0 / (2.0 - lam * lam), rel=1e-15)
    # from w_1 on, the schedule falls towards the paper's constant momentum, 1 + eta, and never passes it
    eta = (1.0 - math.sqrt(1.0 - lam * lam)) / (1.0 + math.sqrt(1.0 - lam * lam))
    assert all(a >= b for a, b in zip(opt.omega[1:], opt.omega[2:]))
    assert opt.omega[-1] >= 1.0 + eta - 1e-15
    assert opt.omega[-1] - (1.0 + eta) < opt.omega[1] - (1.0 + eta)
    plain = DeTAG(LeastSquares([nx.cycle_graph(N)], seed=0), "cpu", _conf(gossip_steps=8, accelerate=False))
    assert plain.omega == [1.0] * 8 and plain.lam == opt.lam


@pytest.mark.parametrize("graph", [nx.complete_graph(5), nx.empty_graph(1)], ids=["complete", "one_node"])
def test_lambda_is_zero_on_the_complete_graph_and_one_node(graph):
    opt = DeTAG(LeastSquares([graph], seed=0), "cpu", _conf(gossip_steps=4))
    assert opt.lam < 1e-15 if graph.number_of_nodes() > 1 else opt.lam == 0.0
    assert np.allclose(opt.omega, 1.0, rtol=0, atol=1e-14)


def _gossip(X, W, omega):
    """One multi-step gossip call through the PyTorch ops: every node local, all rows of W."""
    Wt = torch.as_tensor(W)
    x, xp = X, None
    for om in omega:
        x, xp = ref.ag_gossip(x, xp, Wt, om), x
    return x


@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [10, 32])
def test_one_gossip_call_contracts_at_the_chebyshev_rate(N, K):
    """Applied to the centering matrix, one call of K sub-steps has operator norm max_i |p_K(lambda_i)| on the
    disagreement: exactly 1 / T_K(1 / lambda) for the cycle, below plain gossip's lambda^K for K >= 2.  A random X
    contracts at most that much and keeps its node mean."""
    W = metropolis(nx.cycle_graph(N))
    lam = _cycle_lambda(N)
    omega = ref.chebyshev_weights(ref.mixing_lambda(W), K)
    P = torch.eye(N, dtype=torch.float64) - 1.0 / N
    cheb = torch.linalg.matrix_norm(_gossip(P, W, omega), ord=2).item()
    plain = torch.linalg.matrix_norm(_gossip(P, W, [1.0] * K), ord=2).item()
    bound = do.contraction_bound(lam, K)
    print(f"\nN = {N}, K = {K}: plain {plain:.3f}, Chebyshev {cheb:.3f}, 1/T_K(1/lam) {bound:.3f}")
    assert cheb <= bound + 1e-12 and cheb == pytest.approx(bound, rel=1e-9)
    assert plain == pytest.approx(lam ** K, rel=1e-9)
    if K >= 2:
        assert cheb < plain
    X = torch.as_tensor(np.random.default_rng(N + K).standard_normal((N, 33)))
    Xn = _gossip(X, W, omega)
    dis = lambda A: (A - A.mean(0)).norm().item()          # noqa: E731
    assert dis(Xn) <= bound * dis(X) + 1e-12
    torch.testing.assert_close(Xn.mean(0), X.mean(0), rtol=0, atol=1e-14)


def test_worst_case_factors_of_the_design_table():
    """The plain and Chebyshev worst-case factors quoted in the module docstring's reasoning and DESIGN §2.13."""
    table = {(10, 2): (0.762, 0.615), (10, 4): (0.580, 0.233), (32, 1): (0.987, 0.987), (32, 4): (0.950, 0.823),
             (32, 8): (0.902, 0.513)}
    for (N, K), (plain, cheb) in table.items():
        lam = _cycle_lambda(N)
        assert round(lam ** K, 3) == plain and round(do.contraction_bound(lam, K), 3) == cheb, (N, K)


# --------------------------------------------------------------------------------------------- invariants ----
@ACC
@pytest.mark.parametrize("graph", ["cycle", "wheel", "binary_tree"])
def test_tracker_sum_equals_gradient_sum_every_round(graph, accelerate):
    pr = LeastSquares([GRAPHS[graph]], seed=5)
    opt = DeTAG(pr, "cpu", _conf(gossip_steps=3, accelerate=accelerate))
    for k in range(20):
        opt.run_rounds(1)
        ys, gs = opt.y.sum(0), opt.g_old.sum(0)
        assert (ys - gs).abs().max().item() <= 1e-13 * max(1.0, opt.g_old.abs().max().item()), f"round {k}"


@ACC
def test_one_gossip_step_is_dsgt(accelerate):
    """K = 1: theta = sum_j W_ij (theta_j - alpha y_j) and the tracker are DSGT's (init_grads false), to rounding (z is
    rounded once before the mix)."""
    alpha, R = 0.05, 300
    g = GRAPHS["random"]
    a = DeTAG(LeastSquares([g], seed=2), "cpu", _conf(alpha=alpha, gossip_steps=1, accelerate=accelerate,
                                                      outer_iterations=R))
    b = DSGT(LeastSquares([g], seed=2), "cpu", {"alg_name": "dsgt", "alpha": alpha, "init_grads": False,
                                                "outer_iterations": R})
    diff, scale = [0.0, 0.0], [0.0, 0.0]
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        for q, (got, want) in enumerate(((a.arena.theta, b.arena.theta), (a.y, b.y))):
            diff[q] = max(diff[q], (got - want).norm().item())
            scale[q] = max(scale[q], want.norm().item())
    worst = max(d / s for d, s in zip(diff, scale))
    print(f"\nDeTAG K=1 vs DSGT over {R} rounds: worst relative difference {worst:.2e}")
    assert worst < 1e-12


@ACC
@pytest.mark.parametrize("K", [1, 2, 4])
def test_detag_reaches_the_global_least_squares_solution_where_dsgd_does_not(K, accelerate):
    """Heterogeneous least squares, full deterministic gradients, cycle, constant step: DeTAG converges to the minimiser
    of sum_i f_i; DSGD stops a measurable distance away."""
    rounds, alpha = 2000, 0.02
    pr = LeastSquares([nx.cycle_graph(8)], seed=3)
    opt = DeTAG(pr, "cpu", _conf(alpha=alpha, gossip_steps=K, accelerate=accelerate, outer_iterations=rounds))
    opt.run_rounds(rounds)
    err = np.abs(_np(opt.arena.theta) - pr.solution()).max()
    pd = LeastSquares([nx.cycle_graph(8)], seed=3)
    od = DSGD(pd, "cpu", {"alg_name": "dsgd", "alpha0": alpha, "mu": 0.0, "outer_iterations": rounds})
    od.run_rounds(rounds)
    err_dsgd = np.abs(_np(od.arena.theta) - pd.solution()).max()
    print(f"\nK = {K}, accelerate {accelerate}: max |theta - x*| DeTAG {err:.2e}, DSGD {err_dsgd:.2e}")
    assert err < 1e-10
    assert err_dsgd > 1e-3


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "detag", "alpha": 0.01, "gossip_steps": 2, "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["detag"] is DeTAG
    c = validate_optimizer(dict(BASE))
    assert c["accelerate"] is True and c["profile"] is False
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, accelerate=False, gossip_steps=1, profile=True))


@pytest.mark.parametrize("key", ["alpha", "gossip_steps", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})


@pytest.mark.parametrize("ks", [0, -1, 2.0, 1.5, "2", True])
def test_gossip_steps_must_be_an_integer_at_least_one(ks):
    with pytest.raises(ConfigError, match="gossip_steps"):
        validate_optimizer(dict(BASE, gossip_steps=ks))
    with pytest.raises(ValueError, match="gossip_steps"):
        DeTAG(LeastSquares([GRAPHS["cycle"]]), "cpu", _conf(gossip_steps=ks))


@pytest.mark.parametrize("alpha", [0.0, -0.1, float("inf"), float("nan"), "0.1", True])
def test_alpha_must_be_finite_and_positive(alpha):
    with pytest.raises(ConfigError, match="alpha"):
        validate_optimizer(dict(BASE, alpha=alpha))
    if not isinstance(alpha, (str, bool)):
        with pytest.raises(ValueError, match="alpha"):
            DeTAG(LeastSquares([GRAPHS["cycle"]]), "cpu", _conf(alpha=alpha))


@pytest.mark.parametrize("acc", ["yes", 1, None])
def test_accelerate_must_be_a_bool(acc):
    with pytest.raises(ConfigError, match="accelerate"):
        validate_optimizer(dict(BASE, accelerate=acc))
    with pytest.raises(ValueError, match="accelerate"):
        DeTAG(LeastSquares([GRAPHS["cycle"]]), "cpu", _conf(accelerate=acc))


@pytest.mark.parametrize("key", ["mu", "local_steps", "init_grads", "gamma"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"detag takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        DeTAG(LeastSquares([GRAPHS["cycle"]]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        DeTAG(LeastSquares([GRAPHS["cycle"]]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'detag'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        DeTAG(LeastSquares([nx.cycle_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())


def test_link_drop_fault_injection_is_refused():
    conf = _conf(outer_iterations=4)
    pr = _mnist_problem(conf)
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 4}
    with pytest.raises(ValueError, match="fault_injection"):
        DeTAG(pr, "cpu", copy.deepcopy(conf))


def test_a_changing_graph_is_refused():
    """A problem whose graph changes during the run (the switching sequence) is refused at the first changed round."""
    opt = DeTAG(LeastSquares(ED_GRAPHS["switching"], seed=0), "cpu", _conf())
    with pytest.raises(ValueError, match="fixed graph"):
        opt.run_rounds(3)


def test_a_planned_sequence_of_several_topologies_is_refused():
    """A plan of more than one topology over the run (as the moving online-density plan) is refused before round 0."""
    opt = DeTAG(LeastSquares([nx.cycle_graph(6)], seed=0), "cpu", _conf())
    opt.pr.plan_graphs = lambda oits, k0, dpr, init_draws=0, refresh=True: [nx.cycle_graph(6), nx.path_graph(6)] * oits
    with pytest.raises(ValueError, match="planned graph sequence"):
        opt.run_rounds(1)


# ------------------------------------------------------------------------------------------------ runners ----
def test_detag_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_detag.yaml"), "mnist")
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [(o["alg_name"], o.get("gossip_steps"), o.get("accelerate")) for o in ocs] == [
        ("dsgt", None, None), ("detag", 2, False), ("detag", 2, True)]
    assert all(o["alpha"] == 0.005 for o in ocs)
    paper = load_experiment(os.path.join(EXP, "dist_mnist_local_steps.yaml"), "mnist")
    assert dict(conf["experiment"], name=None) == dict(paper["experiment"], name=None)
    assert conf["problem_configs"]["problem1"] == paper["problem_configs"]["problem2"]


def test_mnist_runner_on_the_detag_yaml(tmp_path, monkeypatch):
    """The three problems of the YAML at a tiny size; DeTAG draws one batch per round, as DSGT does after its initial
    draw."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_detag.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_detag"))
    assert len(out) == 1
    res = {}
    for name in ("dsgt", "detag_k2_plain", "detag_k2"):
        res[name] = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert all(torch.isfinite(v).all() for v in res[name]["validation_loss"])
    fp = {k: [int(torch.as_tensor(v).sum()) for v in r["forward_pass_count"]] for k, r in res.items()}
    assert fp["detag_k2"] == fp["detag_k2_plain"]


def test_density_runner_runs_detag(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="detag")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "detag", "alpha": 0.01, "gossip_steps": 3, "outer_iterations": 4}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "detag_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@ACC
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, accelerate):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha=0.02, gossip_steps=3, accelerate=accelerate, outer_iterations=6)
    full = _mnist_problem(conf)
    of = DeTAG(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = DeTAG(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = DeTAG(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3
    for name in ("y", "g_old", "z"):
        assert torch.equal(getattr(o2, name), getattr(o1, name)), name
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in ("y", "g_old", "z"):
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt


# ------------------------------------------------------------------------------------------ protocol model ----
def test_every_gossip_sub_step_is_a_safe_protocol_round():
    """Each sub-step is one round of the explorer in ``tests/test_protocol_model.py``: announce, wait for the
    neighbors, read parity p & 1, write parity (p + 1) & 1, all in one kernel.  Two gradient rounds at K = 2 are four
    such rounds on the fixed graph; with the waits the engine uses there (no second wait on a static undirected graph,
    the announcement at the round's start) every interleaving of three ranks on a cycle reads the rows of its own round
    and none deadlocks."""
    from test_protocol_model import _sym, explore
    cycle = _sym(3, [(0, 1), (1, 2), (2, 0)])
    v, d, n = explore([cycle] * 4, 3, wait_prev=False, announce_at_start=True, max_states=300_000)
    assert v is None and d is None and n < 300_000
