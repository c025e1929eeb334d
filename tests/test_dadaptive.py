"""Decentralized AMSGrad / AdaGrad on the PyTorch path (CPU): the float64 oracle round by round (with and without the
gossiped second moment), the tracking invariant, the separation from the own-second-moment variant on heterogeneous
least squares, configuration, the runners and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import dadaptive_oracle as do
from test_exact_diffusion import GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.optimizers import ALGORITHMS, DAdaptive
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
VARIANT = pytest.mark.parametrize("variant", ["amsgrad", "adagrad"])
TRACKING = pytest.mark.parametrize("tracking", [True, False], ids=["tracked", "own"])


def _conf(**kw):
    return dict({"alg_name": "dadaptive", "alpha": 0.05, "variant": "amsgrad", "tracking": True,
                 "outer_iterations": 50}, **kw)


def _np(t, n=5):
    return None if t is None else t[:, :n].double().numpy().copy()


# ------------------------------------------------------------------------------------------------ oracle ----
@VARIANT
@TRACKING
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "isolated", "switching"])
def test_torch_path_matches_float64_oracle_round_by_round(graph, tracking, variant):
    pr = LeastSquares(GRAPHS[graph], seed=1)
    extra = {"beta2": 0.99} if variant == "amsgrad" else {}
    opt = DAdaptive(pr, "cpu", _conf(variant=variant, tracking=tracking, beta1=0.8, eps=1e-6, **extra))
    theta = _np(opt.arena.theta)
    st = do.init_state(pr.N, 5, 1e-6, variant, tracking)
    for k in range(12):
        opt.run_rounds(1)
        W = metropolis(GRAPHS[graph][(k + 1) % len(GRAPHS[graph])])
        theta, st = do.round_(theta, st, k=k, W=W, grad_fn=pr.grad, alpha=0.05, beta1=0.8, beta2=0.99, eps=1e-6,
                              variant=variant, tracking=tracking)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        for name in ("m", "v", "vhat", "ut"):
            if st[name] is None:
                assert getattr(opt, name) is None
            else:
                np.testing.assert_allclose(_np(getattr(opt, name)), st[name], rtol=1e-12, atol=1e-15,
                                           err_msg=f"round {k}: {name}")


@VARIANT
@TRACKING
def test_link_drops_match_the_oracle_on_the_dropped_graphs(variant, tracking):
    """Link drops change the graph every round: the oracle walks the graph each round actually used, from the rows
    before the round and the gradients the round drew."""
    conf = _conf(alpha=0.002, variant=variant, tracking=tracking, outer_iterations=6)
    pr = _mnist_problem(conf)
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 6}
    pr._init_faults()
    opt = DAdaptive(pr, "cpu", copy.deepcopy(conf))
    n = pr.layout.n
    graphs = set()
    for k in range(6):
        th0 = _np(pr.arena.theta, n)
        st0 = {name: _np(getattr(opt, name), n) for name in ("m", "v", "vhat", "ut")}
        opt.run_rounds(1)
        W = pr.topology().W
        graphs.add(W.tobytes())
        x = do.wmix(th0, W)
        z = do.wmix(st0["ut"], W) if tracking else None
        g = _np(pr.arena.grad, n)
        step, m, v, vhat, ut = do.update(g, st0["m"], st0["v"], st0["vhat"], z, k=k, alpha=0.002, beta1=0.9,
                                         beta2=0.999, eps=1e-8, variant=variant)
        np.testing.assert_allclose(_np(pr.arena.theta, n), x - step, rtol=1e-5, atol=1e-6, err_msg=f"round {k}")
        np.testing.assert_allclose(_np(opt.vhat, n), vhat, rtol=1e-5, atol=1e-12, err_msg=f"round {k}")
        if tracking:          # fp32 rows: u~ = z + (vhat' - vhat) is held to the magnitudes it is made of
            scale = np.abs(z) + np.abs(vhat) + np.abs(st0["vhat"])
            assert (np.abs(_np(opt.ut, n) - ut) <= 1e-5 * scale + 1e-12).all(), f"round {k}"
    assert len(graphs) > 2


# --------------------------------------------------------------------------------------------- invariants ----
@VARIANT
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete", "random", "switching"])
def test_tracker_sum_equals_second_moment_sum_every_round(graph, variant):
    """sum_i u~_i = sum_i vhat_i after every round (doubly stochastic W, changing graphs too).  Each round adds at most
    a few roundings per node on the magnitudes involved, so the drift is bounded by 64 N u (sum |u~| + sum |vhat|)
    per round, accumulated over the rounds."""
    pr = LeastSquares(GRAPHS[graph], seed=5)
    opt = DAdaptive(pr, "cpu", _conf(variant=variant))
    u = np.finfo(np.float64).eps / 2
    bound = 0.0
    for k in range(40):
        opt.run_rounds(1)
        ut, vh = opt.ut.double(), opt.vhat.double()
        bound += 64 * pr.N * u * (ut.abs().sum(0) + vh.abs().sum(0)).max().item()
        gap = (ut.sum(0) - vh.sum(0)).abs().max().item()
        assert gap <= bound, f"round {k}: {gap:.3e} > {bound:.3e}"


class ScaledLeastSquares(LeastSquares):
    """Heterogeneous least squares whose node objectives are scaled geometrically, 100x from the first to the last
    node: f_i = s_i 0.5 / m |A_i x - b_i|^2.  ``solution()`` is the minimiser of sum_i f_i."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.s = 100.0 ** (np.arange(self.N) / (self.N - 1))
        self._s = torch.as_tensor(self.s, dtype=self._A.dtype).view(-1, 1)

    def grad(self, i, x):
        return self.s[i] * super().grad(i, x)

    def solution(self):
        H = sum(self.s[i] * self.A[i].T @ self.A[i] for i in range(self.N))
        r = sum(self.s[i] * self.A[i].T @ self.b[i] for i in range(self.N))
        return np.linalg.solve(H, r)

    def batched_grads(self, views):
        loss = super().batched_grads(views)
        for i in range(self.N):
            views[i][0].mul_(self.s[i])
        return loss * self._s


def _mean_error(variant, tracking, alpha, rounds):
    pr = ScaledLeastSquares([nx.cycle_graph(8)], seed=3)
    opt = DAdaptive(pr, "cpu", _conf(variant=variant, tracking=tracking, alpha=alpha, outer_iterations=rounds))
    opt.run_rounds(rounds)
    xs = pr.solution()
    return np.linalg.norm(_np(opt.arena.theta).mean(0) - xs) / np.linalg.norm(xs)


@VARIANT
def test_tracking_reaches_the_global_minimiser_where_the_own_second_moment_does_not(variant):
    """8-node cycle, full gradients, node scales spread 100x, alpha 0.01 for 5000 rounds: with the tracker the node
    mean ends within 1e-2 (relative) of the minimiser of sum_i f_i; dividing by each node's own second moment stops
    more than 0.3 away.  The tracked error falls with the step: a 3x smaller step over the same alpha * rounds ends
    closer."""
    tracked = _mean_error(variant, True, 0.01, 5000)
    own = _mean_error(variant, False, 0.01, 5000)
    small = _mean_error(variant, True, 0.01 / 3, 15000)
    print(f"\n{variant}: relative error of the node mean: tracked {tracked:.2e}, own {own:.2e}, "
          f"tracked at alpha / 3 {small:.2e}")
    assert tracked < 1e-2
    assert own > 0.3
    assert small < tracked


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "dadaptive", "alpha": 0.01, "variant": "amsgrad", "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["dadaptive"] is DAdaptive
    c = validate_optimizer(dict(BASE))
    assert (c["tracking"], c["beta1"], c["beta2"], c["eps"], c["update_graph"], c["profile"]) == (
        True, 0.9, 0.999, 1e-8, True, False)
    c = validate_optimizer(dict(BASE, variant="adagrad"))
    assert "beta2" not in c and c["tracking"] is True
    for key in ("alpha", "variant", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in BASE.items() if k != key})
    for key in ("update_graph", "consensus_backend", "checkpoint_every", "resume"):
        validate_optimizer(dict(BASE, **{key: True}))
    validate_optimizer(dict(BASE, tracking=False, beta1=0.0, beta2=0.0, eps=1e-3))


def test_unknown_variant_is_refused():
    for v in ("adam", "AMSGrad", None):
        with pytest.raises(ConfigError, match="variant must be one of amsgrad|adagrad"):
            validate_optimizer(dict(BASE, variant=v))
    with pytest.raises(ValueError, match="variant"):
        DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(variant="adam"))


def test_out_of_range_alpha_is_refused():
    for alpha in (0.0, -0.1, "0.1", True):
        with pytest.raises(ConfigError, match="alpha must be > 0"):
            validate_optimizer(dict(BASE, alpha=alpha))
    with pytest.raises(ValueError, match="alpha"):
        DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(alpha=0.0))


@pytest.mark.parametrize("key", ["beta1", "beta2"])
def test_out_of_range_beta_is_refused(key):
    for b in (1.0, -0.1, 1.5, "0.9", True):
        with pytest.raises(ConfigError, match=rf"{key} must be in \[0, 1\)"):
            validate_optimizer(dict(BASE, **{key: b}))
    with pytest.raises(ValueError, match=key):
        DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(**{key: 1.0}))


def test_tracking_must_be_a_bool():
    for t in ("yes", 1, None):
        with pytest.raises(ConfigError, match="tracking must be true or false"):
            validate_optimizer(dict(BASE, tracking=t))


def test_beta2_with_adagrad_is_refused():
    with pytest.raises(ConfigError, match="beta2 applies to variant amsgrad only"):
        validate_optimizer(dict(BASE, variant="adagrad", beta2=0.999))
    with pytest.raises(ValueError, match="beta2"):
        DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(variant="adagrad", beta2=0.99))


def test_non_positive_or_infinite_eps_is_refused():
    for eps in (0.0, -1e-8, float("inf"), float("nan"), "1e-8"):
        with pytest.raises(ConfigError, match="eps must be finite and > 0"):
            validate_optimizer(dict(BASE, eps=eps))
    with pytest.raises(ValueError, match="eps"):
        DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(eps=0.0))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order: dadaptive runs the synchronous 'jacobi' order only"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'dadaptive'"):
        validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        DAdaptive(LeastSquares([nx.cycle_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")


def test_adaptive_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_adaptive.yaml"), "mnist")
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [(o["alg_name"], o.get("variant"), o.get("tracking")) for o in ocs] == [
        ("dsgd", None, None), ("dadaptive", "amsgrad", False), ("dadaptive", "amsgrad", True),
        ("dadaptive", "adagrad", True)]
    ed = load_experiment(os.path.join(EXP, "dist_mnist_hetero_ed.yaml"), "mnist")
    assert dict(conf["experiment"], name=None) == dict(ed["experiment"], name=None)
    assert conf["problem_configs"]["problem1"] == ed["problem_configs"]["problem3"]


@pytest.mark.parametrize("variant", ["amsgrad", "adagrad"])
def test_checkpoint_carries_the_variant_rows(variant):
    for tracking in (True, False):
        opt = DAdaptive(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(variant=variant, tracking=tracking))
        want = {"m", "vhat"} | ({"v"} if variant == "amsgrad" else set()) | ({"ut"} if tracking else set())
        assert set(opt.STATE) == want
        assert set(opt.state_dict()) == want | {"k", "theta"}
        assert (opt.vhat == 1e-8).all() and (opt.m == 0).all()
        if tracking:
            assert (opt.ut == 1e-8).all()


# ------------------------------------------------------------------------------------------------ runners ----
def test_mnist_runner_on_the_adaptive_yaml(tmp_path, monkeypatch):
    """All four problems of the new YAML at a tiny size through the MNIST runner."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_adaptive.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_adaptive"))
    assert len(out) == 1
    for name in ("dsgd", "amsgrad_own", "amsgrad_tracked", "adagrad_tracked"):
        res = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert len(res["validation_loss"]) == 2
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])


def test_mnist_template_runs_dadaptive(tmp_path, monkeypatch):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True, use_cuda=False)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="dadaptive")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = dict(BASE, variant="adagrad", outer_iterations=5)
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))[0]
    res = torch.load(os.path.join(out, "dadaptive_results.pt"), weights_only=False)
    assert len(res["validation_loss"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


def test_density_runner_runs_dadaptive(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="dadaptive")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = dict(BASE, outer_iterations=4)
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "dadaptive_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@VARIANT
@TRACKING
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, variant, tracking):
    """AdaGrad's running mean divides by the round count, which the checkpoint's k restores."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha=0.002, variant=variant, tracking=tracking, outer_iterations=6)
    full = _mnist_problem(conf)
    of = DAdaptive(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = DAdaptive(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = DAdaptive(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3
    for name in o2.STATE:
        assert torch.equal(getattr(o2, name), getattr(o1, name)), name
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for name in o2.STATE:
        assert torch.equal(getattr(o2, name), getattr(of, name)), name
    assert second.forward_cnt == full.forward_cnt
