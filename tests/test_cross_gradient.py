"""Cross-gradient gossip on the PyTorch path (CPU, float64): the NumPy oracle round by round on six graph kinds, at three
cross weights and two network sizes; the properties of the method (D-PSGD at cross_weight 0, local SGD on the edgeless
graph, centralized SGD on the complete graph, the gradient sum at consensus, the smaller heterogeneity bias on least
squares, the cross point at the own row); every configuration refusal; the runners and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import hsgd_oracle as ho
import xg_oracle as xo
from test_exact_diffusion import LeastSquares, _mnist_problem, _synthetic
from test_gt_hsgd import LSProblem
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, CrossGradient, GossipPGA
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


def _random(N, p, seed):
    for s in range(seed, seed + 1000):
        g = nx.gnp_random_graph(N, p, seed=s)
        if nx.is_connected(g):
            return g
    raise AssertionError("no connected graph")


def _graphs(N):
    return {"cycle": nx.cycle_graph(N), "path": nx.path_graph(N), "star": nx.star_graph(N - 1),
            "complete": nx.complete_graph(N), "random": _random(N, 0.4, 3),
            "binary_tree": nx.convert_node_labels_to_integers(nx.balanced_tree(2, 3).subgraph(range(N)))}


GRAPHS4, GRAPHS12 = _graphs(4), _graphs(12)
LAMS = [0.0, 0.3, 1.0]


def _conf(**kw):
    return dict({"alg_name": "cross_gradient", "alpha0": 0.05, "mu": 0.0, "cross_weight": 0.5,
                 "outer_iterations": 50}, **kw)


def _np(t, n=5):
    return t[:, :n].double().numpy().copy()


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("N", [4, 12])
@pytest.mark.parametrize("lam", LAMS)
@pytest.mark.parametrize("graph", sorted(GRAPHS4))
def test_torch_path_matches_float64_oracle_round_by_round(graph, lam, N):
    """Six graph kinds at 4 and 12 nodes (one and several ranks' worth), minibatches of 8 rows, a decaying step."""
    R = 8
    g = (GRAPHS4 if N == 4 else GRAPHS12)[graph]
    assert g.number_of_nodes() == N
    pr = LSProblem(g, batch=8, seed=1)
    conf = _conf(cross_weight=lam, mu=0.5, outer_iterations=R)
    opt = CrossGradient(pr, "cpu", conf)
    alphas = opt.alpha_table(R)
    want = xo.run(_np(pr.arena.theta), ho.metropolis(g), lam, alphas, pr.batch_grad, R)
    for k, theta in enumerate(want):
        opt.run_rounds(1)
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-11, atol=1e-11, err_msg=f"round {k}")
    assert pr.calls.tolist() == [R] * pr.N
    assert opt.alph == alphas[-1]


# ------------------------------------------------------------------------------------------- properties ----
def _dpsgd_round(pr, alpha):
    """D-PSGD on the PyTorch ops: the gradient at the published row, then the mixed row minus the step."""
    a = pr.arena
    topo = pr.topology()
    xmix = ref.dsgd_mix(pr.gather_rows(a.theta), torch.as_tensor(topo.W, dtype=a.dtype))
    pr.compute_grads()
    a.theta.copy_(xmix)
    ref.dsgd_step_(a.theta, a.grad, alpha)


@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_cross_weight_zero_is_dpsgd_bit_for_bit(model):
    """Property 1: lam = 0 gives d = 1 g + sum 0 g' = g, so every round is D-PSGD's, bit for bit."""
    R = 6
    conf = _conf(cross_weight=0.0, mu=0.3, outer_iterations=R)
    if model == "mnist":
        pa, pb = _mnist_problem(conf), _mnist_problem(conf)
    else:
        pa, pb = LSProblem(GRAPHS4["random"], batch=8, seed=2), LSProblem(GRAPHS4["random"], batch=8, seed=2)
    opt = CrossGradient(pa, "cpu", conf)
    for k, alpha in enumerate(opt.alpha_table(R)):
        opt.run_rounds(1)
        _dpsgd_round(pb, alpha)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"
    assert pa.forward_cnt == pb.forward_cnt and (pa.calls == pb.calls).all()


@pytest.mark.parametrize("lam", [0.0, 0.5, 1.0])
def test_edgeless_graph_is_local_sgd_bit_for_bit(lam):
    """Property 2: with no edge W_ii = 1, xmix = x and d = g: Gossip-PGA's local SGD (gossip false, period past the
    run), i.e. N independent SGD runs, bit for bit."""
    R = 8
    pa, pb = LSProblem(nx.empty_graph(5), batch=8, seed=3), LSProblem(nx.empty_graph(5), batch=8, seed=3)
    a = CrossGradient(pa, "cpu", _conf(cross_weight=lam, mu=0.2, outer_iterations=R))
    b = GossipPGA(pb, "cpu", {"alg_name": "gossip_pga", "alpha0": 0.05, "mu": 0.2, "period": R + 1, "gossip": False,
                              "outer_iterations": R})
    assert a.coef0.tolist() == [1.0] * 5
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"


def test_complete_graph_full_weight_is_centralized_minibatch_sgd():
    """Property 3: complete graph, lam = 1, equal starting rows: every node steps along (1/N) sum_j grad f_j(x; xi_j),
    the nodes stay equal to round-off and the run is minibatch SGD on the union of the N minibatches."""
    R, N, alpha = 10, 6, 0.05
    pr = LSProblem(nx.complete_graph(N), batch=8, seed=4)
    pr.arena.theta.copy_(pr.arena.theta[:1].expand_as(pr.arena.theta))
    opt = CrossGradient(pr, "cpu", _conf(cross_weight=1.0, alpha0=alpha, outer_iterations=R))
    x = _np(pr.arena.theta)[0]
    for k in range(R):
        opt.run_rounds(1)
        x = x - alpha * pr.batch_grad(np.repeat(x[None], N, axis=0), k).mean(0)
        th = _np(pr.arena.theta)
        assert np.abs(th - th[:1]).max() <= 1e-13 * np.abs(th).max(), f"round {k}"
        np.testing.assert_allclose(th, np.repeat(x[None], N, axis=0), rtol=1e-12, atol=1e-12, err_msg=f"round {k}")


@pytest.mark.parametrize("lam", [0.3, 1.0])
@pytest.mark.parametrize("graph", ["cycle", "star", "random", "binary_tree"])
def test_gradient_sum_at_consensus(graph, lam):
    """Property 4: with every row equal, sum_i d_i = sum_i g_ii for a doubly stochastic W (sum_i c0_i g_i + sum_i sum_j
    lam W_ij g_j(x) = sum_i (1 - lam + lam sum_j W_ji) g_i)."""
    pr = LSProblem(GRAPHS12[graph], batch=8, seed=5)
    pr.arena.theta.copy_(pr.arena.theta[:1].expand_as(pr.arena.theta))
    opt = CrossGradient(pr, "cpu", _conf(cross_weight=lam, outer_iterations=2))
    seen = []
    step = ref.xg_step_

    def spy(theta, xmix, grad, recv, coef0, coef, alpha):
        seen.append((grad.clone(), step(theta, xmix, grad, recv, coef0, coef, alpha)))
        return seen[-1][1]
    ref.xg_step_ = spy
    try:
        opt.run_rounds(1)
    finally:
        ref.xg_step_ = step
    g, d = seen[0]
    gs, ds = g.sum(0), d.sum(0)
    assert (ds - gs).abs().max().item() <= 1e-13 * g.abs().sum(0).max().item()


def test_full_weight_lowers_the_heterogeneity_bias_on_least_squares():
    """Property 5: heterogeneous least squares with full-batch gradients on the 8-node cycle.  The fixed point of the
    affine round map at lam = 1 lies strictly closer to the minimiser of sum_i f_i than the one at lam = 0 (D-PSGD), at
    the same step; and the PyTorch path converges to the lam = 1 fixed point."""
    alpha, N = 0.02, 8
    pr = LSProblem(nx.cycle_graph(N), seed=3)
    x_star = pr.solution()
    H = np.stack([2.0 * pr.A[i].T @ pr.A[i] / pr.A.shape[1] for i in range(N)])
    r = np.stack([2.0 * pr.A[i].T @ pr.b[i] / pr.A.shape[1] for i in range(N)])
    W = ho.metropolis(pr.graph)
    dist = {lam: np.linalg.norm(xo.fixed_point(H, r, W, lam, alpha) - x_star[None]) for lam in (0.0, 1.0)}
    print(f"\n|x_fp - x*| at alpha {alpha}: lam 0 {dist[0.0]:.4e}, lam 1 {dist[1.0]:.4e}")
    assert dist[1.0] < dist[0.0]
    rounds = 1500
    opt = CrossGradient(pr, "cpu", _conf(cross_weight=1.0, alpha0=alpha, outer_iterations=rounds))
    opt.run_rounds(rounds)
    np.testing.assert_allclose(_np(opt.arena.theta), xo.fixed_point(H, r, W, 1.0, alpha), rtol=0, atol=1e-8)


@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_cross_point_at_the_own_row_gives_the_own_gradient(model):
    """Property 6 on the autograd path: a cross point equal to the node's row gives g_ii exactly, on the same draw."""
    if model == "mnist":
        pr = _mnist_problem(_conf())
    else:
        pr = LSProblem(GRAPHS4["cycle"], batch=8, seed=6)
    pr.count_draws_all(3)
    calls, fwd = pr.calls.copy(), pr.forward_cnt
    P = 3
    points = pr.arena.theta.unsqueeze(0).repeat(P, 1, 1)
    grads = torch.zeros_like(points)
    pr.compute_grads_multi(points, grads)
    assert (pr.calls == calls + 1).all() and pr.forward_cnt == fwd + pr.train_batch_size
    for p in range(P):
        assert torch.equal(grads[p], pr.arena.grad), p


def test_compute_grads_multi_takes_every_point_on_one_draw():
    """Different points, one draw: each slot's gradient is autograd's at that point on the indices of the draw."""
    pr = LSProblem(GRAPHS4["path"], batch=8, seed=7)
    pr.count_draws_all(2)
    calls = pr.calls.copy()
    g = torch.Generator().manual_seed(0)
    points = pr.arena.theta.unsqueeze(0) + torch.randn((2,) + tuple(pr.arena.theta.shape), generator=g,
                                                       dtype=pr.dtype)
    points[..., pr.n:] = 0
    grads = torch.zeros_like(points)
    pr.compute_grads_multi(points, grads)
    x = np.stack([_np(points[p]) for p in range(2)])
    for p in range(2):
        full = np.zeros((pr.N, 5))
        for i in range(pr.N):
            idx = pr.schedules[i].indices(int(calls[i]), pr.seed, i).numpy()
            A, b = pr.A[i][idx], pr.b[i][idx]
            full[i] = 2.0 * A.T @ (A @ x[p, i] - b) / len(idx)
        np.testing.assert_allclose(_np(grads[p]), full, rtol=1e-12, atol=1e-12)


def test_gradient_evaluations_and_cross_points():
    pr = LSProblem(nx.star_graph(4), batch=8, seed=8)
    opt = CrossGradient(pr, "cpu", _conf())
    assert opt.dmax == 4 and opt.grad_evals() == (5 + 2 * 4, 5 * 5)
    assert pr.xg_grad_evals == {"useful_per_round": 13, "launched_per_round": 25, "rounds": 50}
    assert opt.coef0[0].item() == 0.5 + 0.5 * (1 - 4 / 5)
    tx = ref.xg_cross_points(pr.arena.theta, opt._src_node, opt._live, 0)
    assert torch.equal(tx[:, 0], pr.arena.theta[1:5])                         # the hub sees every leaf
    assert torch.equal(tx[0, 1:], pr.arena.theta[[0] * 4])                     # a leaf sees the hub in slot 0
    assert torch.equal(tx[1:, 1:], pr.arena.theta[1:5].unsqueeze(0).expand(3, 4, -1))   # and itself in idle slots


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "cross_gradient", "alpha0": 0.01, "cross_weight": 0.5, "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["cross_gradient"] is CrossGradient
    c = validate_optimizer(dict(BASE))
    assert c["mu"] == 0.0 and c["profile"] is False
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, cross_weight=0, mu=0.001, profile=True))
    validate_optimizer(dict(BASE, cross_weight=1.0))


@pytest.mark.parametrize("key", ["alpha0", "cross_weight", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})


@pytest.mark.parametrize("w", [-0.1, 1.5, float("inf"), float("nan"), "0.5", True])
def test_cross_weight_must_be_finite_and_in_zero_one(w):
    with pytest.raises(ConfigError, match="cross_weight"):
        validate_optimizer(dict(BASE, cross_weight=w))
    with pytest.raises(ValueError, match="cross_weight"):
        CrossGradient(LSProblem(GRAPHS4["cycle"]), "cpu", _conf(cross_weight=w))


@pytest.mark.parametrize("key", ["alpha0", "mu"])
def test_step_schedule_must_be_finite_and_nonnegative(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer(dict(BASE, **{key: -1.0}))
    with pytest.raises(ValueError, match=key):
        CrossGradient(LSProblem(GRAPHS4["cycle"]), "cpu", _conf(**{key: float("nan")}))


@pytest.mark.parametrize("key", ["alpha", "beta", "gamma", "period", "gossip"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"cross_gradient takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        CrossGradient(LSProblem(GRAPHS4["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        CrossGradient(LSProblem(GRAPHS4["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'cross_gradient'"):
        validate_experiment(conf, "mnist")
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 4}
    validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        CrossGradient(LSProblem(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())


def test_link_drops_are_refused():
    conf = _exp("cycle")
    pc = conf["problem_configs"]["problem1"]
    pc["optimizer_config"] = dict(BASE)
    validate_experiment(copy.deepcopy(conf), "mnist")
    pc["fault_injection"] = {"link_drop_prob": 0.2, "seed": 1}
    with pytest.raises(ConfigError, match="fault_injection: cross_gradient needs a fixed graph"):
        validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="fault_injection"):
        CrossGradient(LSProblem(GRAPHS4["cycle"], faults={"link_drop_prob": 0.2, "seed": 1}), "cpu", _conf())


class _TwoGraphs(LSProblem):
    def plan_graphs(self, oits, k0, draws_per_round, init_draws=0, refresh=True):
        return [self.graph if k % 2 == 0 else nx.path_graph(self.N) for k in range(oits)]


def test_a_planned_sequence_of_more_than_one_topology_is_refused():
    opt = CrossGradient(_TwoGraphs(GRAPHS4["cycle"]), "cpu", _conf(outer_iterations=4))
    with pytest.raises(ValueError, match="cross_gradient needs a fixed graph"):
        opt.run_rounds(1)


def test_the_online_density_runner_is_refused():
    from nn_distributed_training_b200.utils.config import validate_problem
    pc = {"problem_name": "p", "train_batch_size": 8, "val_batch_size": 8, "metrics": ["validation_loss"],
          "metrics_config": {"evaluate_frequency": 2}, "comm_radius": 1.0, "optimizer_config": dict(BASE)}
    validate_problem(copy.deepcopy(pc), "problem_configs.p", "density")
    with pytest.raises(ConfigError, match="online-density runner moves the graph"):
        validate_problem(pc, "problem_configs.p", "online_density")


def test_reference_api_problem_is_refused():
    """A problem behind the reference API draws its minibatch inside local_batch_loss and cannot replay it."""
    with pytest.raises(ValueError, match="same minibatch"):
        CrossGradient(LeastSquares([nx.cycle_graph(6)]), "cpu", _conf())


def test_a_degree_past_the_wait_capacity_is_refused():
    """The round-start wait has one thread per in-neighbor, 256 of them: a hub of degree 257 is refused."""
    with pytest.raises(ValueError, match="257 in-neighbors"):
        CrossGradient(LSProblem(nx.star_graph(257), m=2, batch=2), "cpu", _conf())


# ------------------------------------------------------------------------------------------------ runners ----
def test_cross_gradient_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_cross_gradient.yaml"), "mnist")
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [(o["alg_name"], o.get("cross_weight")) for o in ocs] == [("dsgd", None), ("cross_gradient", 0.0),
                                                                     ("cross_gradient", 1.0)]
    assert all(o["alpha0"] == 0.005 and o["mu"] == 0.001 for o in ocs)
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    keep = ("data_split_type", "graph", "model", "loss")
    assert {k: conf["experiment"][k] for k in keep} == {k: paper["experiment"][k] for k in keep}


def test_mnist_runner_writes_the_gradient_evaluations(tmp_path, monkeypatch):
    """The three problems of the YAML at a tiny size: every arm draws one batch per round, and the cross-gradient arms
    write xg_grad_evals (N + 2|E| useful, N (1 + dmax) launched per round) into their results."""
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_cross_gradient.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_cross_gradient"))
    assert len(out) == 1
    res = {name: torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
           for name in ("dsgd", "cross_gradient_w0", "cross_gradient_w1")}
    for r in res.values():
        assert all(torch.isfinite(v).all() for v in r["validation_loss"])
    assert "xg_grad_evals" not in res["dsgd"]
    for name in ("cross_gradient_w0", "cross_gradient_w1"):
        assert res[name]["xg_grad_evals"] == {"useful_per_round": 4 + 8, "launched_per_round": 4 * 3, "rounds": 3}
    fp = {k: [int(torch.as_tensor(v).sum()) for v in r["forward_pass_count"]] for k, r in res.items()}
    assert fp["cross_gradient_w0"] == fp["cross_gradient_w1"] == fp["dsgd"]


def test_density_runner_writes_the_gradient_evaluations(tmp_path):
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
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="cross_gradient")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "cross_gradient", "alpha0": 0.01, "cross_weight": 1.0, "outer_iterations": 4}
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "cross_gradient_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])
    ev = res["xg_grad_evals"]
    assert ev["rounds"] == 4 and 3 <= ev["useful_per_round"] <= ev["launched_per_round"]


# ------------------------------------------------------------------------------------------------ resume ----
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, cross_weight=0.7, outer_iterations=6)
    full = _mnist_problem(conf)
    of = CrossGradient(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = CrossGradient(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = CrossGradient(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and o2.alph == o1.alph
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert second.forward_cnt == full.forward_cnt
