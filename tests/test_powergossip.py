"""PowerGossip on the PyTorch path (CPU): the matrix table, the start vectors, the float64 oracle of
``tests/powergossip_oracle.py`` round by round in both phases, sum conservation, bit-equal endpoint vectors and a
non-increasing consensus distance at alpha = 0, the exact removal of a rank-one difference, the DSGD equivalence for
1-D parameters, a zero difference keeping its vector, the refusals, configuration, the runners and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import consensus_oracle as co
import powergossip_oracle as po
from test_exact_diffusion import LeastSquares, _synthetic
from test_relaysum import _mnist_problem
from test_sgp import _exp
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.models.fourier_nn import FourierNet
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, PowerGossip
from nn_distributed_training_b200.parallel.arena import FlatLayout
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer
from nn_distributed_training_b200.utils.graph_generation import Topology

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


def _random():
    for seed in range(1000):
        g = nx.gnp_random_graph(7, 0.45, seed=seed)
        if nx.is_connected(g):
            return g
    raise AssertionError


GRAPHS = {"cycle": nx.cycle_graph(5), "path": nx.path_graph(5), "star": nx.star_graph(5), "wheel": nx.wheel_graph(6),
          "complete": nx.complete_graph(4), "random": _random()}


def _conf(**kw):
    return dict({"alg_name": "powergossip", "alpha0": 0.05, "mu": 0.0, "gamma": 0.8, "outer_iterations": 40}, **kw)


class Layers(torch.nn.Module):
    def __init__(self, dtype):
        super().__init__()
        self.w1 = torch.nn.Parameter(torch.zeros(4, 3, dtype=dtype))
        self.b1 = torch.nn.Parameter(torch.zeros(4, dtype=dtype))
        self.w2 = torch.nn.Parameter(torch.zeros(2, 3, 2, dtype=dtype))
        self.b2 = torch.nn.Parameter(torch.zeros(2, dtype=dtype))


class Quadratic:
    """Node i minimises 0.5 |theta - t_i|^2 over matrices and biases (``Layers``): gradient theta - t_i, different
    minimisers per node."""

    capturable_grads = False

    def __init__(self, graph, seed=0, dtype=torch.float64, module=Layers):
        rng = np.random.default_rng(seed)
        self.graph = graph
        self.N = graph.number_of_nodes()
        torch.manual_seed(seed)
        self.models = [module(dtype) for _ in range(self.N)]
        with torch.no_grad():
            for m in self.models:
                for p in m.parameters():
                    p.copy_(torch.as_tensor(rng.standard_normal(tuple(p.shape)), dtype=dtype))
        self.targets = [[torch.as_tensor(rng.standard_normal(tuple(p.shape)), dtype=dtype) for p in m.parameters()]
                        for m in self.models]
        self.conf = {"metrics_config": {"evaluate_frequency": 10 ** 9}}

    def update_graph(self):
        pass

    def batched_grads(self, views):
        for i in range(self.N):
            for v, p, t in zip(views[i], self.models[i].parameters(), self.targets[i]):
                v.copy_(p.detach() - t)
        return torch.zeros(self.N, 1, dtype=views[0][0].dtype)

    def evaluate_metrics(self, at_end=False):
        pass


def _rows(opt):
    return opt.arena.theta.double().numpy().copy()


def _cd(rows):
    return float(((rows - rows.mean(0)) ** 2).sum())


def _endpoints(opt):
    t = opt.topo
    rs = t.reverse_slots()
    for i, nb in enumerate(t.neighbors_noself):
        for e, j in enumerate(nb):
            assert torch.equal(opt.vec[i, e], opt.vec[j, rs[i][e]]), f"edge ({i}, {j})"


# ---------------------------------------------------------------------------------------------- layout ----
def test_matrix_table_of_the_paper_conv_net():
    lay = ref.PgLayout(FlatLayout.from_module(MNISTConvNet(3, 5, 64)))
    assert [(m, n) for _, m, n, _, _ in lay.mats] == [(3, 25), (64, 432), (10, 64)]
    assert (lay.P, lay.Q, lay.B) == (77, 521, 77)
    assert (lay.msg_len(0), lay.msg_len(1)) == (154, 598) and lay.width == 600
    assert [sg[1] for sg in lay.vecs] == [3, 64, 10]


def test_matrix_table_of_a_fourier_net():
    net = FourierNet([2, 32, 16, 1])
    layout = FlatLayout.from_module(net)
    lay = ref.PgLayout(layout)
    for s, sg in zip(layout.slots, lay.segs):
        assert sg[0] == s.offset
        if len(s.shape) >= 2:
            assert (sg[1], sg[2]) == (s.shape[0], int(np.prod(s.shape[1:])))
        else:
            assert sg[2] == 0 and sg[1] == s.numel
    assert lay.P == sum(sg[1] for sg in lay.mats) and lay.Q == sum(sg[2] for sg in lay.mats)
    assert lay.width % 4 == 0 and lay.width >= max(lay.msg_len(0), lay.msg_len(1))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_start_vectors_are_unit_and_shared_by_both_endpoints(dtype):
    opt = PowerGossip(Quadratic(GRAPHS["wheel"], dtype=dtype), "cpu", _conf())
    _endpoints(opt)
    lay = opt.lay
    for i, nb in enumerate(opt.topo.neighbors_noself):
        for e in range(len(nb)):
            for _, m, n, poff, qoff in lay.mats:
                for v in (opt.vec[i, e, poff: poff + m], opt.vec[i, e, lay.P + qoff: lay.P + qoff + n]):
                    assert abs(float(v.double().norm()) - 1.0) < 4 * torch.finfo(dtype).eps
    assert torch.equal(ref.pg_start_vectors(lay, 1, 2, dtype), opt.vec[2, opt.topo.neighbors_noself[2].index(1)])


# ---------------------------------------------------------------------------------------------- oracle ----
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(name):
    g = GRAPHS[name]
    pr = Quadratic(g, seed=1)
    opt = PowerGossip(pr, "cpu", _conf(mu=0.5))
    t = Topology(g)
    nbrs, rs, lay = t.neighbors_noself, t.reverse_slots(), opt.lay
    alphas = opt.alpha_table(8)
    u = co.unit_roundoff(np.float64)
    for k in range(8):
        theta, vec, msg = _rows(opt), opt.vec.double().numpy().copy(), opt.msg.double().numpy().copy()
        x, ex, vn, ev = po.mix(theta, vec, msg, nbrs, rs, t.W, opt.gamma, lay.segs, lay.P, lay.Q, k & 1, u)
        grad = x - _targets(opt, pr)
        opt.run_rounds(1)
        h, eh, out, eo = po.step(x, grad, 0.0, alphas[k], vn, np.zeros_like(msg), nbrs, lay.segs,
                                 lay.P, lay.Q, (k + 1) & 1, u)
        co.check(f"round {k} theta", _rows(opt), h, eh + ex, 16)
        co.check(f"round {k} vec", opt.vec.numpy(), vn, ev, 16)
        co.check(f"round {k} msg", opt.msg.numpy(), out, eo + np.abs(out) * 1e-12, 16)


def _targets(opt, pr):
    """The rows of the nodes' minimisers (zero in the layout's holes)."""
    out = np.zeros((pr.N, opt.arena.n_pad))
    for i in range(pr.N):
        for s, t in zip(opt.arena.layout.slots, pr.targets[i]):
            out[i, s.offset: s.offset + s.numel] = t.reshape(-1).numpy()
    return out


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_every_round_conserves_the_sum_and_never_spreads_the_nodes(name, dtype):
    """alpha = 0, gamma = 1: sum_i theta_i stays put to rounding, both endpoints hold the same vector bits and the
    consensus distance never increases, in both phases."""
    pr = Quadratic(GRAPHS[name], seed=2, dtype=dtype)
    opt = PowerGossip(pr, "cpu", _conf(alpha0=0.0, gamma=1.0))
    tol = 64 * torch.finfo(dtype).eps
    s0, prev = _rows(opt).sum(0), _cd(_rows(opt))
    for k in range(10):
        opt.run_rounds(1)
        rows = _rows(opt)
        assert np.abs(rows.sum(0) - s0).max() <= tol * (1 + np.abs(rows).sum()), f"round {k}"
        _endpoints(opt)
        c = _cd(rows)
        assert c <= prev * (1 + tol), f"round {k}: {c} > {prev}"
        prev = c


def test_phase_one_removes_a_rank_one_difference_exactly():
    """Two nodes whose matrices differ by a b^T: round 0 (phase 0) finds p = +-a / |a|, round 1 (phase 1) projects the
    whole difference, and at gamma = 1 both nodes land on the midpoint (the biases too)."""
    pr = Quadratic(nx.path_graph(2), seed=3)
    rng = np.random.default_rng(4)
    with torch.no_grad():
        for p0, p1 in zip(pr.models[0].parameters(), pr.models[1].parameters()):
            if p0.dim() >= 2:
                m = p0.shape[0]
                n = p0.numel() // m
                p1.copy_(p0 + torch.as_tensor(np.outer(rng.standard_normal(m), rng.standard_normal(n))).reshape(p0.shape))
    opt = PowerGossip(pr, "cpu", _conf(alpha0=0.0, gamma=1.0))
    mid = _rows(opt).mean(0)
    opt.run_rounds(2)
    rows = _rows(opt)
    np.testing.assert_allclose(rows[0], mid, rtol=0, atol=1e-13)
    np.testing.assert_allclose(rows[1], mid, rtol=0, atol=1e-13)


class VecModel(torch.nn.Module):
    def __init__(self, dtype):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.zeros(5, dtype=dtype))


class VecLeastSquares(LeastSquares):
    """``LeastSquares`` with a 1-D parameter: nothing to compress."""

    def __init__(self, graphs, seed=0):
        super().__init__(graphs, seed=seed)
        old = self.models
        self.models = [VecModel(torch.float64) for _ in range(self.N)]
        with torch.no_grad():
            for a, b in zip(self.models, old):
                a.weight.copy_(b.weight.reshape(-1))

    def batched_grads(self, views):
        x = torch.stack([m.weight.detach() for m in self.models])
        r = torch.einsum("imn,in->im", self._A, x) - self._b
        g = torch.einsum("imn,im->in", self._A, r) / self.m
        for i in range(self.N):
            views[i][0].copy_(g[i])
        return 0.5 * (r * r).mean(1, keepdim=True)


@pytest.mark.parametrize("name", ["cycle", "star", "random"])
def test_one_dimensional_parameters_at_gamma_one_are_dsgd(name):
    g = GRAPHS[name]
    a, b = VecLeastSquares([g], seed=5), VecLeastSquares([g], seed=5)
    oa = PowerGossip(a, "cpu", _conf(gamma=1.0, mu=0.5))
    ob = DSGD(b, "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": 40})
    assert oa.lay.P == oa.lay.Q == 0 and oa.vec.shape[-1] == 0
    for k in range(30):
        oa.run_rounds(1)
        ob.run_rounds(1)
        np.testing.assert_allclose(_rows(oa), _rows(ob), rtol=1e-12, atol=1e-12, err_msg=f"round {k}")


def test_a_zero_difference_keeps_the_stored_vector():
    pr = Quadratic(nx.path_graph(2), seed=6)
    with torch.no_grad():
        for p0, p1 in zip(pr.models[0].parameters(), pr.models[1].parameters()):
            p1.copy_(p0)
    opt = PowerGossip(pr, "cpu", _conf(alpha0=0.0))
    before = opt.vec.clone()
    opt.run_rounds(2)
    assert torch.equal(opt.vec, before)
    assert torch.equal(opt.arena.theta[0], opt.arena.theta[1])


# ---------------------------------------------------------------------------------------------- refusals ----
def test_a_directed_graph_is_refused():
    with pytest.raises(ValueError, match="undirected"):
        PowerGossip(Quadratic(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())
    conf = _exp("directed_cycle")
    conf["problem_configs"]["problem1"]["optimizer_config"] = _conf(outer_iterations=3)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'powergossip'"):
        validate_experiment(conf, "mnist")


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order: powergossip runs the synchronous 'jacobi' order only"):
        validate_optimizer(_conf(mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        PowerGossip(Quadratic(nx.cycle_graph(4)), "cpu", _conf(mixing_order="reference"))


def test_link_drop_fault_injection_is_refused():
    pr = _mnist_problem(_conf(), graph=nx.cycle_graph(4))
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 0, "to_round": 6}
    pr._init_faults()
    with pytest.raises(ValueError, match="link-drop fault_injection"):
        PowerGossip(pr, "cpu", _conf())


def test_a_multi_topology_plan_is_refused():
    pr = _mnist_problem(_conf(), graph=nx.cycle_graph(4))
    pr.plan_graphs = lambda oits, k0, dpr, init_draws=0, refresh=True: [nx.cycle_graph(4), nx.star_graph(3)] * oits
    opt = PowerGossip(pr, "cpu", _conf())
    with pytest.raises(ValueError, match="powergossip needs a fixed graph"):
        opt.train()


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "powergossip", "alpha0": 0.01, "gamma": 0.5, "outer_iterations": 3}


def test_registered_and_config_keys():
    assert ALGORITHMS["powergossip"] is PowerGossip
    c = validate_optimizer(dict(BASE))
    assert c["mu"] == 0.0 and c["profile"] is False
    for key in ("alpha0", "gamma", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in BASE.items() if k != key})
    for key in ("profile", "consensus_backend", "checkpoint_every", "checkpoint_dir", "resume"):
        validate_optimizer(dict(BASE, **{key: "fused" if key == "consensus_backend" else 1}))
    for key in ("rank", "compressor", "beta", "alpha"):
        with pytest.raises(ConfigError, match=f"powergossip takes no key '{key}'"):
            validate_optimizer(dict(BASE, **{key: 1}))


@pytest.mark.parametrize("gamma", [0.0, -0.5, 1.5, float("inf"), float("nan"), "0.5", True])
def test_gamma_outside_zero_one_is_refused(gamma):
    with pytest.raises(ConfigError, match="gamma must be finite and in"):
        validate_optimizer(dict(BASE, gamma=gamma))


def test_alpha0_and_mu_are_checked():
    validate_optimizer(dict(BASE, alpha0=0.0, gamma=1.0))
    with pytest.raises(ConfigError, match="alpha0 must be finite and >= 0"):
        validate_optimizer(dict(BASE, alpha0=-0.1))
    with pytest.raises(ConfigError, match="mu must be finite and >= 0"):
        validate_optimizer(dict(BASE, mu=-1.0))


def test_the_yaml_is_the_paper_setup_with_three_arms():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_powergossip.yaml"), "mnist")
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    for key in ("model", "data_split_type", "graph"):
        assert conf["experiment"][key] == paper["experiment"][key]
    ocs = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [o["alg_name"] for o in ocs] == ["dsgd", "choco_sgd", "powergossip"]
    assert ocs[1]["compressor"] == "topk" and ocs[1]["topk_ratio"] == 0.01
    assert {o["alpha0"] for o in ocs} == {0.005} and {o["outer_iterations"] for o in ocs} == {2000}


def test_checkpoint_carries_the_vectors_and_the_messages():
    opt = PowerGossip(Quadratic(GRAPHS["star"]), "cpu", _conf())
    assert opt.STATE == ("vec", "msg") and opt.msg.shape == (6, 5, opt.lay.width)
    assert set(opt.state_dict()) == {"k", "theta", "vec", "msg", "alph"}


# ------------------------------------------------------------------------------------------------ runners ----
def test_mnist_runner_on_the_powergossip_yaml(tmp_path, monkeypatch):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_powergossip.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_powergossip"))
    assert len(out) == 1
    for name in ("dsgd", "choco_topk", "powergossip"):
        res = torch.load(os.path.join(out[0], f"{name}_results.pt"), weights_only=False)
        assert len(res["validation_loss"]) == 2
        assert all(torch.isfinite(v).all() for v in res["validation_loss"])


def test_density_runner_runs_powergossip(tmp_path):
    from test_runners import _small_density_conf, _write, synthetic_dir  # noqa: F401
    from nn_distributed_training_b200.experiments import dist_dense_ex
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path / "floor")
    os.makedirs(d)
    write_dataset(d, n_paths=4, seed=0)
    conf = _small_density_conf("dist_dense_v2.yaml", d, tmp_path)
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 3}
    conf["experiment"]["individual_training"]["train_solo"] = False
    pc = conf["problem_configs"]["problem1"]
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="powergossip")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = dict(BASE, outer_iterations=4)
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "powergossip_results.pt"), weights_only=False)
    assert len(res["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path):
    """The checkpoint after round 3 resumes in phase 1: the vectors and messages come back bit for bit."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, outer_iterations=6)
    g = nx.cycle_graph(4)
    full = _mnist_problem(conf, graph=g)
    of = PowerGossip(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf, graph=g)
    o1 = PowerGossip(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf, graph=g)
    o2 = PowerGossip(second, "cpu", copy.deepcopy(conf))
    assert not torch.equal(o2.vec, o1.vec)
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and o2.alph == o1.alph
    assert torch.equal(o2.vec, o1.vec) and torch.equal(o2.msg, o1.msg)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert torch.equal(o2.vec, of.vec) and torch.equal(o2.msg, of.msg)
    assert second.forward_cnt == full.forward_cnt
