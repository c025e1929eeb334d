"""DP-DSGD and DECOR on the PyTorch path (CPU, float64): the Philox known-answer vectors of the noise stream's host twin,
the accountant against closed forms, the NumPy oracle round by round, DSGD bit for bit with a clip above every norm and
no noise, the network sum of the pairwise noise, the noise covariance, every configuration refusal, the runners with
the ``privacy`` record and checkpoint/resume with the ledger."""
import copy
import glob
import math
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import dp_oracle as do
from test_exact_diffusion import _mnist_problem, _synthetic
from test_gt_hsgd import GRAPHS, LSProblem, _np
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, DPDSGD
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
DROPS = {"link_drop_prob": 0.3, "seed": 5, "from_round": 2, "to_round": 12}


def _conf(**kw):
    return dict({"alg_name": "dp_dsgd", "alpha0": 0.05, "mu": 0.5, "clip_norm": 1.0, "noise_multiplier": 0.3,
                 "pair_noise_multiplier": 0.5, "outer_iterations": 50}, **kw)


def _alphas(alpha0, mu, n):
    out, a = [], alpha0
    for _ in range(n):
        a = a * (1.0 - mu * a)
        out.append(a)
    return out


def _zero_grads(pr):
    """theta = 0, g = 0: a round with alpha = 1 leaves theta = -v."""
    pr.arena.theta.zero_()

    def compute_grads():
        pr.arena.grad.zero_()
        return pr.last_losses
    pr.compute_grads = compute_grads


# ------------------------------------------------------------------------------------------- noise stream ----
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
], ids=["zeros", "ones", "pi"])
def test_philox_twin_reproduces_the_random123_known_answers(ctr, key, want):
    got = ref.philox4x32_10(np.array([ctr], dtype=np.uint64), key)[0]
    assert [int(x) for x in got] == list(want)


def test_normals_are_standard_and_the_streams_are_distinct():
    key = ref.dp_key(3)
    x = ref.dp_normals(key, 0, 2, ref.DP_LOCAL, 1 << 16)
    n = x.size
    assert abs(x.mean()) < 5 / math.sqrt(n) and abs(x.var() - 1) < 5 * math.sqrt(2 / n)
    assert np.array_equal(x, ref.dp_normals(key, 0, 2, ref.DP_LOCAL, 1 << 16))
    for other in (ref.dp_normals(key, 1, 2, ref.DP_LOCAL, 64), ref.dp_normals(key, 0, 1, 2, 64),
                  ref.dp_normals(ref.dp_key(4), 0, 2, ref.DP_LOCAL, 64)):
        assert not np.array_equal(x[:64], other)
    # the stream of an element pair does not depend on the row length
    assert np.array_equal(ref.dp_normals(key, 5, 0, 1, 64), ref.dp_normals(key, 5, 0, 1, 256)[:64])


# ------------------------------------------------------------------------------------------- accountant ----
def test_accountant_on_the_complete_graph():
    N, zd, zp = 10, 1.3, 0.7
    eav, allo = ref.dp_rho(np.ones((N, N)) / N, zd, zp)
    want = do.complete_inverse_diagonal(N, zd, zp)
    assert abs(want - 0.195742159) < 1e-9
    np.testing.assert_allclose(eav, 2 * want, rtol=1e-13)
    np.testing.assert_allclose(allo, 2 / zd ** 2, rtol=0)


@pytest.mark.parametrize("N", [3, 10, 17])
def test_accountant_on_the_cycle(N):
    from hsgd_oracle import metropolis
    eav, _ = ref.dp_rho(metropolis(nx.cycle_graph(N)), 0.8, 2.5)
    np.testing.assert_allclose(eav, 2 * do.cycle_inverse_diagonal(N, 0.8, 2.5), rtol=1e-12)


def test_accountant_limits():
    from hsgd_oracle import metropolis
    W = metropolis(nx.cycle_graph(10))
    eav, allo = ref.dp_rho(W, 1.1, 0.0)            # no pair noise: both guarantees are the local one
    np.testing.assert_allclose(eav, allo, rtol=1e-14)
    eav, allo = ref.dp_rho(W, 1.1, 1e4)            # pair noise without bound: at most a factor N
    np.testing.assert_allclose(eav, 2 / (10 * 1.1 ** 2), rtol=1e-6)
    np.testing.assert_allclose(allo, 2 / 1.1 ** 2, rtol=0)
    eav, allo = ref.dp_rho(W, 0.0, 3.0)            # no local noise: no guarantee, reported as inf
    assert np.isinf(eav).all() and np.isinf(allo).all()
    assert ref.dp_epsilon(eav, 1e-5) == math.inf
    rho = np.array([0.5, 2.0])
    assert ref.dp_epsilon(rho, 1e-5) == pytest.approx(2.0 + 2 * math.sqrt(2.0 * math.log(1e5)), rel=1e-15)


def test_ledger_on_a_link_drop_run_is_the_sum_over_the_rounds_graphs():
    R = 12
    pr = LSProblem(GRAPHS["wheel"], batch=8, seed=1, faults=DROPS)
    graphs = pr.plan_graphs(R, 0, 1)
    assert len({tuple(sorted(g.edges())) for g in graphs}) > 3
    opt = DPDSGD(pr, "cpu", _conf(outer_iterations=R))
    opt.run_rounds(R)
    from hsgd_oracle import metropolis
    want = sum(ref.dp_rho(metropolis(g), 0.3, 0.5)[0] for g in graphs)
    np.testing.assert_allclose(opt.rho_eav, want, rtol=1e-12)
    np.testing.assert_allclose(opt.rho_all, R * 2 / 0.3 ** 2, rtol=1e-13)
    assert (opt.rho_eav < opt.rho_all).all()


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("zs", [(0.0, 0.0), (0.3, 0.0), (0.3, 0.5), (0.0, 0.5)], ids=["clip", "ldp", "decor", "pair"])
@pytest.mark.parametrize("drops", [False, True], ids=["static", "link_drops"])
@pytest.mark.parametrize("graph", ["cycle", "star", "random", "complete"])
def test_torch_path_matches_float64_oracle_round_by_round(graph, drops, zs):
    R = 12
    pr = LSProblem(GRAPHS[graph], batch=8, seed=1, faults=DROPS if drops else None)
    graphs = pr.plan_graphs(R, 0, 1)
    opt = DPDSGD(pr, "cpu", _conf(clip_norm=2.0, noise_multiplier=zs[0], pair_noise_multiplier=zs[1],
                                  outer_iterations=R, noise_seed=9))
    n_pad = pr.arena.n_pad
    live = ref.choco_live(pr.arena.layout).numpy()

    def grad(x, k):
        g = np.zeros_like(x)
        g[:, :5] = pr.batch_grad(x[:, :5], k)
        return g
    want = do.run(pr.arena.theta.numpy(), graphs, _alphas(0.05, 0.5, R), 2.0, zs[0], zs[1], ref.dp_key(9), grad, R, live)
    for k, theta in enumerate(want):
        opt.run_rounds(1)
        np.testing.assert_allclose(pr.arena.theta.numpy(), theta, rtol=1e-11, atol=1e-11, err_msg=f"round {k}")
    assert (pr.arena.theta.numpy()[:, 5:] == 0).all() and n_pad > 5      # the padding stays 0


@pytest.mark.parametrize("model", ["least_squares", "mnist"])
def test_clip_above_every_norm_and_no_noise_is_dsgd_bit_for_bit(model):
    R = 8
    pconf = _conf(clip_norm=1e30, noise_multiplier=0.0, pair_noise_multiplier=0.0, outer_iterations=R)
    dconf = {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": R}
    if model == "mnist":
        pa, pb = _mnist_problem(pconf), _mnist_problem(dconf)
    else:
        pa, pb = (LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS),
                  LSProblem(GRAPHS["random"], batch=8, seed=2, faults=DROPS))
    a, b = DPDSGD(pa, "cpu", pconf), DSGD(pb, "cpu", dconf)
    for k in range(R):
        a.run_rounds(1)
        b.run_rounds(1)
        assert torch.equal(pa.arena.theta, pb.arena.theta), f"round {k}"
        assert a.alph == b.alph
    assert pa.forward_cnt == pb.forward_cnt and (pa.calls == pb.calls).all()


def test_clipping_bounds_every_step():
    """alpha0 = 1, no noise and no mixing (the edgeless graph): every step moves theta by exactly min(||g||, C)."""
    R, C = 5, 0.05
    pr = LSProblem(nx.empty_graph(4), batch=8, seed=3)
    opt = DPDSGD(pr, "cpu", _conf(alpha0=1.0, mu=0.0, clip_norm=C, noise_multiplier=0.0, pair_noise_multiplier=0.0,
                                  outer_iterations=R))
    for k in range(R):
        before = pr.arena.theta.clone()
        g = pr.batch_grad(_np(before), k)
        opt.run_rounds(1)
        step = (before - pr.arena.theta).norm(dim=1).numpy()
        np.testing.assert_allclose(step, np.minimum(np.linalg.norm(g, axis=1), C), rtol=1e-12)


@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete"])
def test_pairwise_noise_cancels_over_the_network(graph):
    """z_dp = 0, theta = 0, g = 0, alpha = 1: after one round theta_i = -v_i, and sum_i v_i = 0 to float64 rounding
    (each edge's normal enters once with each sign)."""
    pr = LSProblem(GRAPHS[graph], n=300, batch=8, seed=4)
    _zero_grads(pr)
    opt = DPDSGD(pr, "cpu", _conf(alpha0=1.0, mu=0.0, clip_norm=1.5, noise_multiplier=0.0, pair_noise_multiplier=2.0,
                                  outer_iterations=3))
    opt.run_rounds(1)
    v = -pr.arena.theta.numpy()
    assert np.abs(v).max() > 1.0
    dmax = max(d for _, d in GRAPHS[graph].degree())
    bound = 4 * dmax * np.abs(v).max() * 2.0 ** -52
    assert np.abs(v.sum(0)).max() <= bound, (np.abs(v.sum(0)).max(), bound)


def test_noise_covariance_matches_the_accountants_sigma():
    """The empirical node-by-node covariance of v over the elements of 8 rounds matches C^2 (z_dp^2 I + z_pair^2 Lap)
    at a fixed seed.  Each entry of the sample covariance of n Gaussian samples has standard deviation
    sqrt((S_ii S_jj + S_ij^2) / n); every entry must lie within 5 of them."""
    N, C, zd, zp = 8, 1.5, 0.7, 0.9
    g = nx.cycle_graph(N)
    g.add_edge(0, 4)
    pr = LSProblem(g, n=2000, batch=8, seed=5)
    opt = DPDSGD(pr, "cpu", _conf(clip_norm=C, noise_multiplier=zd, pair_noise_multiplier=zp, outer_iterations=8))
    topo = pr.topology()
    live = ref.choco_live(pr.arena.layout).numpy()
    V = np.concatenate([opt.noise_rows(k, topo).numpy()[:, live] for k in range(8)], axis=1)
    n = V.shape[1]
    emp = V @ V.T / n
    lap = nx.laplacian_matrix(g, nodelist=range(N)).toarray().astype(np.float64)
    S = C * C * (zd * zd * np.eye(N) + zp * zp * lap)
    sd = np.sqrt((np.outer(np.diag(S), np.diag(S)) + S * S) / n)
    z = np.abs(emp - S) / sd
    print(f"\nworst |emp - Sigma| / sd over the 8 x 8 entries: {z.max():.2f} (n = {n})")
    assert z.max() < 5.0


# ------------------------------------------------------------------------------------------------ config ----
BASE = {"alg_name": "dp_dsgd", "alpha0": 0.01, "clip_norm": 1.0, "noise_multiplier": 0.5, "outer_iterations": 3}


def test_registered_and_config_defaults():
    assert ALGORITHMS["dp_dsgd"] is DPDSGD
    c = validate_optimizer(dict(BASE))
    assert c["mu"] == 0.0 and c["pair_noise_multiplier"] == 0.0 and c["target_delta"] == 1e-5
    assert c["update_graph"] is True and c["profile"] is False and "noise_seed" not in c
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, alpha0=0.0, mu=0.1, noise_multiplier=0, pair_noise_multiplier=3.0, target_delta=0.5,
                            noise_seed=-4, update_graph=False, profile=True))
    pr = LSProblem(GRAPHS["cycle"], seed=6)
    opt = DPDSGD(pr, "cpu", _conf())
    assert opt.noise_seed == 6 and opt.delta == 1e-5 and opt.key == ref.dp_key(6)


@pytest.mark.parametrize("key", ["alpha0", "clip_norm", "noise_multiplier", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})


@pytest.mark.parametrize("key,bad", [
    ("mu", -0.5), ("mu", float("inf")), ("mu", float("nan")),
    ("alpha0", -0.1), ("alpha0", float("inf")), ("alpha0", float("nan")), ("alpha0", True),
    ("clip_norm", 0.0), ("clip_norm", -1.0), ("clip_norm", float("inf")), ("clip_norm", "1"),
    ("noise_multiplier", -0.5), ("noise_multiplier", float("nan")), ("noise_multiplier", False),
    ("pair_noise_multiplier", -1.0), ("pair_noise_multiplier", float("inf")),
    ("target_delta", 0.0), ("target_delta", 1.0), ("target_delta", -1e-5), ("target_delta", True),
    ("noise_seed", 1.5), ("noise_seed", "3"), ("noise_seed", True)])
def test_out_of_range_values_are_refused(key, bad):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer(dict(BASE, **{key: bad}))
    with pytest.raises(ValueError, match=key):
        DPDSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(**{key: bad}))


@pytest.mark.parametrize("key", ["clip", "delta", "alpha", "period", "gossip", "beta"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"dp_dsgd takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        DPDSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        DPDSGD(LSProblem(GRAPHS["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'dp_dsgd'"):
        validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        DPDSGD(LSProblem(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())


# ------------------------------------------------------------------------------------------------ runners ----
ARMS = [("dsgd", None, None), ("dp_dsgd", 0.0, 0.0), ("dp_dsgd", "ldp", 0.0), ("dp_dsgd", "decor", "decor")]
NAMES = ["dsgd", "clipped_dsgd", "ldp_dsgd", "decor"]


def test_dp_yaml_validates_and_its_multipliers_give_the_stated_epsilons():
    """The two noisy arms are calibrated to about the same eavesdropper epsilon over the run; the YAML's comment
    states the accountant's values, recomputed here."""
    from hsgd_oracle import metropolis
    conf = load_experiment(os.path.join(EXP, "dist_mnist_dp.yaml"), "mnist")
    pcs = list(conf["problem_configs"].values())
    ocs = [p["optimizer_config"] for p in pcs]
    assert [p["problem_name"] for p in pcs] == NAMES
    assert [o["alg_name"] for o in ocs] == [a[0] for a in ARMS]
    assert ocs[1]["noise_multiplier"] == 0.0 and ocs[1]["pair_noise_multiplier"] == 0.0
    assert ocs[2]["pair_noise_multiplier"] == 0.0 and ocs[3]["pair_noise_multiplier"] > 0.0
    e = conf["experiment"]
    assert e["graph"]["type"] == "cycle" and e["graph"]["num_nodes"] == 10 and e["data_split_type"] == "hetero"
    W = metropolis(nx.cycle_graph(10))
    eps = []
    for o in ocs[2:]:
        rho = o["outer_iterations"] * ref.dp_rho(W, o["noise_multiplier"], o["pair_noise_multiplier"])[0]
        eps.append(ref.dp_epsilon(rho, o["target_delta"]))
    print(f"\neavesdropper epsilon: local DP {eps[0]:.3f}, DECOR {eps[1]:.3f}")
    assert abs(eps[0] - 8.0) < 0.05 and abs(eps[1] - 8.0) < 0.05


def test_mnist_runner_on_the_dp_yaml_writes_the_privacy_record(tmp_path, monkeypatch):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_dp.yaml")) as f:
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
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_dp"))
    assert len(out) == 1
    res = {n: torch.load(os.path.join(out[0], f"{n}_results.pt"), weights_only=False) for n in NAMES}
    assert "privacy" not in res["dsgd"]
    assert all(torch.isfinite(v).all() for r in res.values() for v in r["validation_loss"])
    fp = {n: [int(torch.as_tensor(v).sum()) for v in r["forward_pass_count"]] for n, r in res.items()}
    assert len({tuple(v) for v in fp.values()}) == 1
    for n in NAMES[1:]:
        rec = res[n]["privacy"]
        assert rec["target_delta"] == 1e-5 and rec["rounds"] == 5
        assert rec["rho_eavesdropper"].shape == (4,) and rec["rho_any_observer"].dtype == torch.float64
    assert res["clipped_dsgd"]["privacy"]["epsilon_any_observer"] == math.inf
    ldp, decor = res["ldp_dsgd"]["privacy"], res["decor"]["privacy"]
    assert ldp["epsilon_eavesdropper"] == ldp["epsilon_any_observer"] < math.inf
    assert decor["epsilon_eavesdropper"] < decor["epsilon_any_observer"]


def test_density_runner_runs_dp_dsgd(tmp_path):
    from test_runners import _small_density_conf, _write, synthetic_dir  # noqa: F401
    from nn_distributed_training_b200.experiments import dist_dense_ex
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path / "floor")
    os.makedirs(d)
    write_dataset(d, n_paths=4, seed=0)
    res = {}
    for name, oc in [("dsgd", {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.0, "outer_iterations": 4}),
                     ("clip_off", {"alg_name": "dp_dsgd", "alpha0": 0.01, "clip_norm": 1e30, "noise_multiplier": 0.0,
                                   "outer_iterations": 4}),
                     ("decor", {"alg_name": "dp_dsgd", "alpha0": 0.01, "clip_norm": 1.0, "noise_multiplier": 0.5,
                                "pair_noise_multiplier": 1.0, "outer_iterations": 4})]:
        sub = tmp_path / name
        sub.mkdir()
        conf = _small_density_conf("dist_dense_v2.yaml", d, sub)
        # a fixed graph: the YAML's random graph is drawn from the unseeded global `random` module, so two arms
        # could run on different graphs
        conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 3}
        conf["experiment"]["individual_training"]["train_solo"] = False
        pc = conf["problem_configs"]["problem1"]
        pc.update(train_batch_size=300, val_batch_size=400, problem_name="arm")
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"] = oc
        torch.manual_seed(0)                 # the same initial models in every arm
        np.random.seed(0)
        dist_dense_ex.experiment(_write(str(sub), "d.yaml", conf))
        out = glob.glob(os.path.join(str(sub), "*_dist_dense_v2"))[0]
        res[name] = torch.load(os.path.join(out, "arm_results.pt"), weights_only=False)
    assert len(res["decor"]["mesh_grid_density"]) == 3
    assert all(torch.isfinite(v).all() for v in res["decor"]["validation_loss"])
    # a clip above every norm and no noise is DSGD: the same metrics bit for bit
    assert all(torch.equal(a, b) for a, b in zip(res["dsgd"]["validation_loss"], res["clip_off"]["validation_loss"]))
    assert res["decor"]["privacy"]["epsilon_eavesdropper"] < res["decor"]["privacy"]["epsilon_any_observer"]


def test_privacy_record_hook_belongs_to_the_optimizer_training_the_problem():
    """The problem's ``privacy_record`` hook is the DP optimizer's while it trains the problem; an optimizer built on the
    same problem later resets it, so a results file never carries a stale record.  A foreign problem (reference API,
    wrapped in an adapter) gets no hook: the record stays the optimizer's."""
    from nn_distributed_training_b200.optimizers.base import ReferenceProblemAdapter
    pr = LSProblem(GRAPHS["cycle"], seed=2)
    assert pr.privacy_record is None
    opt = DPDSGD(pr, "cpu", _conf(outer_iterations=2))
    opt.run_rounds(2)
    assert pr.privacy_record == opt.privacy_record and pr.privacy_record()["rounds"] == 2
    DSGD(pr, "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": 2})
    assert pr.privacy_record is None

    class Foreign:
        def __init__(self, inner):
            self.N, self.graph, self.conf = inner.N, inner.graph, inner.conf
            self.models = [inner.models[i] for i in range(inner.N)]

        def update_graph(self):
            pass
    foreign = Foreign(LSProblem(GRAPHS["cycle"], seed=2))
    fo = DPDSGD(foreign, "cpu", _conf(outer_iterations=2, noise_seed=1))
    assert isinstance(fo.pr, ReferenceProblemAdapter) and "privacy_record" not in vars(fo.pr)
    assert not hasattr(foreign, "privacy_record") and fo.privacy_record()["rounds"] == 0


# ------------------------------------------------------------------------------------------------ resume ----
def test_state_round_trip_carries_the_ledger():
    pr = LSProblem(GRAPHS["wheel"], batch=8, seed=1, faults=DROPS)
    opt = DPDSGD(pr, "cpu", _conf(outer_iterations=6))
    opt.run_rounds(3)
    sd = copy.deepcopy(opt.state_dict())
    assert np.array_equal(sd["rho_eav"], opt.rho_eav) and sd["rho_eav"].dtype == np.float64
    fresh = DPDSGD(LSProblem(GRAPHS["wheel"], batch=8, seed=1, faults=DROPS), "cpu", _conf(outer_iterations=6))
    fresh.load_state_dict(sd)
    assert np.array_equal(fresh.rho_eav, opt.rho_eav) and np.array_equal(fresh.rho_all, opt.rho_all)
    assert fresh.k == 3 and fresh.alph == opt.alph


@pytest.mark.parametrize("stop", [3, 4])
def test_checkpoint_resume_is_bit_exact(tmp_path, stop):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, clip_norm=0.5, noise_multiplier=0.01, pair_noise_multiplier=0.02,
                 outer_iterations=8)
    full = _mnist_problem(conf)
    of = DPDSGD(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = DPDSGD(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=stop, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = stop                   # "crash" after round `stop`
    o1.train()
    assert o1.k == stop
    second = _mnist_problem(conf)
    o2 = DPDSGD(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=stop, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == stop and o2.alph == o1.alph and np.array_equal(o2.rho_eav, o1.rho_eav)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt
    assert np.array_equal(o2.rho_eav, of.rho_eav) and np.array_equal(o2.rho_all, of.rho_all)
