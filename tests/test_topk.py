"""Top-k sparsified gossip for CHOCO-SGD and BEER on the PyTorch path (CPU): the code-row layout, the selection rule
against an independent NumPy oracle, the contraction, both optimizers against their float64 oracles, BEER's invariants
and exactness, CHOCO's consensus, ratio 1 against the compressor none, configuration, the runner and checkpoint/resume."""
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
import topk_oracle as tko
from test_exact_diffusion import GRAPHS, LeastSquares, metropolis
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import BEER, DSGD, ChocoSGD
from nn_distributed_training_b200.parallel.arena import FlatLayout, ParamSlot
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
STATIC = {k: v for k, v in GRAPHS.items() if k != "switching"}
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
NPDT = {torch.float32: np.float32, torch.float64: np.float64}
# two slots with an alignment hole and row padding: dead elements that must never be selected
LAYOUT = FlatLayout([ParamSlot("a", (5,), 0, 5), ParamSlot("b", (70,), 8, 70), ParamSlot("c", (100,), 80, 100)])


def _np(t):
    return t.detach().double().cpu().numpy().copy()


def _nbrs(W):
    return [[j for j in range(W.shape[0]) if j != i and W[i, j] != 0] for i in range(W.shape[0])]


def _rows(dtype, L=4, seed=0):
    """Random rows with a spread of magnitudes, and the hard cases: heavy ties (also straddling the threshold), an
    all-zero row, values one ulp apart and -0 against +0.  Dead elements hold large values: they must not be picked."""
    g = torch.Generator().manual_seed(seed)
    live = ref.choco_live(LAYOUT)
    n = LAYOUT.n_pad
    v = torch.randn(L, n, generator=g, dtype=torch.float64) * torch.exp(3 * torch.randn(L, n, generator=g, dtype=torch.float64))
    v = v.to(dtype)
    v[:, ~live] = 1e30
    rows = [v[i] for i in range(L)]
    ties = torch.where(torch.arange(n) % 3 == 0, 2.0, -1.0).to(dtype)          # a third at |v| = 2, the rest at 1
    ties[torch.arange(n) % 7 == 0] = -2.0
    rows.append(ties)
    rows.append(torch.zeros(n, dtype=dtype))
    ulp = torch.full((n,), 1.0, dtype=dtype)
    ulp[1::2] = torch.nextafter(torch.tensor(1.0, dtype=dtype), torch.tensor(2.0, dtype=dtype))
    ulp[2::5] = -ulp[2::5]
    rows.append(ulp)
    z = torch.zeros(n, dtype=dtype)
    z[::2] = -0.0
    z[50] = 3.0
    rows.append(z)
    out = torch.stack(rows)
    out[:, ~live] = 1e30
    return out, live


# ------------------------------------------------------------------------------------------------ format ----
def test_code_bytes_of_the_paper_model():
    """PAPER MNIST (n_pad 28 544, 28 440 parameters): k = 285 at ratio 0.01; 285 (8 + 4) = 3 420 B -> 3 424 in fp64 and
    285 (4 + 4) = 2 280 B -> 2 288 in fp32."""
    lay = FlatLayout.from_module(MNISTConvNet(3, 5, 64))
    live = ref.choco_live(lay)
    assert lay.n_pad == 28544 and int(live.sum()) == 28440
    k = ref.choco_topk_k(0.01, int(live.sum()))
    assert k == 285
    assert ref.choco_code_bytes("topk", lay.n_pad, torch.float64, k) == 3424
    assert ref.choco_code_bytes("topk", lay.n_pad, torch.float32, k) == 2288
    assert ref.choco_topk_k(1e-9, 28440) == 1 and ref.choco_topk_k(1.0, 28440) == 28440
    for bad in (0.0, -0.1, 1.01):
        with pytest.raises(ValueError, match="topk_ratio"):
            ref.choco_topk_k(bad, 100)


@DTYPES
@pytest.mark.parametrize("k", [1, 7, 64, "n_live"])
def test_layout_round_trip_and_selection_against_numpy(k, dtype):
    """Indices ascending, unique and live; values exact; dec(q) = v at the indices; the selection is the NumPy oracle's
    (np.lexsort on (index, -key)) on random rows, heavy ties across the threshold, an all-zero row, last-ulp
    differences and -0 against +0; padding bytes zero."""
    v, live = _rows(dtype)
    n_live = int(live.sum())
    k = n_live if k == "n_live" else k
    codes, dec = ref.choco_encode(v, "topk", live, k)
    nb = ref.choco_code_bytes("topk", LAYOUT.n_pad, dtype, k)
    assert codes.shape == (v.shape[0], nb) and nb % 16 == 0
    assert torch.equal(ref.choco_decode(codes, "topk", LAYOUT.n_pad, dtype, live, k), dec)
    s = v.element_size()
    for r in range(v.shape[0]):
        row = codes[r].numpy()
        d, idx, vals = tko.topk_decode(row, LAYOUT.n_pad, NPDT[dtype], k)
        assert np.all(np.diff(idx.astype(np.int64)) > 0) and live.numpy()[idx].all()
        want = tko.topk_select(v[r].numpy(), live.numpy(), k)
        assert np.array_equal(idx, want), f"row {r}"
        assert np.array_equal(vals.view(np.uint8), v[r].numpy()[idx].view(np.uint8))      # exact, -0 kept
        np.testing.assert_array_equal(d, dec[r].double().numpy())
        assert not row[k * (s + 4):].any()


def test_ties_go_to_the_smaller_index_and_zero_signs_tie():
    live = torch.ones(128, dtype=torch.bool)
    v = torch.zeros(1, 128, dtype=torch.float64)
    v[0, [5, 9, 40, 100]] = torch.tensor([-2.0, 2.0, 2.0, 3.0], dtype=torch.float64)
    assert ref.choco_topk_select(v, live, 3).tolist() == [[5, 9, 100]]
    z = torch.zeros(1, 128, dtype=torch.float32)
    z[0, :10] = -0.0
    assert ref.choco_topk_select(z, live, 4).tolist() == [[0, 1, 2, 3]]
    u = torch.full((1, 128), 1.0, dtype=torch.float32)
    u[0, 77] = torch.nextafter(torch.tensor(1.0), torch.tensor(2.0))
    assert ref.choco_topk_select(u, live, 2).tolist() == [[0, 77]]


@DTYPES
def test_contraction(dtype):
    """|v - Q(v)|^2 <= (1 - k / n_live) |v|^2 on every row, for several k."""
    v, live = _rows(dtype, L=8, seed=3)
    v[:, ~live] = 0
    n_live = int(live.sum())
    for k in (1, 3, 17, 90, n_live):
        _, dec = ref.choco_encode(v, "topk", live, k)
        e2 = ((dec.double() - v.double()) ** 2).sum(1)
        n2 = (v.double() ** 2).sum(1)
        assert torch.all(e2 <= (1 - k / n_live) * n2 * (1 + 1e-12)), k


# ------------------------------------------------------------------------------------------------ oracle ----
def _conf(alg, **kw):
    if alg == "choco_sgd":
        c = {"alg_name": "choco_sgd", "alpha0": 0.05, "mu": 0.5, "gamma": 0.5, "compressor": "topk",
             "topk_ratio": 0.4, "outer_iterations": 50}
    else:
        c = {"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "compressor": "topk", "topk_ratio": 0.4,
             "outer_iterations": 50}
    return dict(c, **kw)


def _dec(code, n_pad, k):
    return np.stack([tko.topk_decode(code[i], n_pad, np.float64, k)[0] for i in range(code.shape[0])])


@pytest.mark.parametrize("graph", sorted(STATIC))
def test_choco_torch_path_matches_float64_oracle_round_by_round(graph):
    pr = LeastSquares(STATIC[graph], seed=1)
    opt = ChocoSGD(pr, "cpu", _conf("choco_sgd"))
    assert opt.topk_k == 2            # ceil(0.4 * 5)
    W = metropolis(STATIC[graph][0])
    nbrs = _nbrs(W)
    n_pad, live, k = opt.arena.n_pad, opt.live.numpy(), opt.topk_k
    theta, x_hat, s = _np(opt.arena.theta), np.zeros((pr.N, n_pad)), np.zeros((pr.N, n_pad))
    code = opt.code.numpy().copy()
    alpha, u = 0.05, 2.0 ** -53
    for r in range(8):
        opt.run_rounds(1)
        alpha = alpha * (1.0 - 0.5 * alpha)
        theta, s, e_th, e_s = cho.mix(theta, x_hat, s, _dec(code, n_pad, k), nbrs, W, 0.5, u, 0.0)
        g = np.zeros_like(theta)
        g[:, :5] = np.stack([pr.grad(i, theta[i, :5]) for i in range(pr.N)])
        theta = theta - alpha * g
        np.testing.assert_allclose(_np(opt.arena.theta), theta, rtol=1e-11, atol=1e-12, err_msg=f"round {r}")
        np.testing.assert_allclose(_np(opt.s), s, rtol=1e-11, atol=1e-12, err_msg=f"round {r}")
        code = opt.code.numpy().copy()
        v = _np(opt.arena.theta) - x_hat
        for i in range(pr.N):      # the published code is the top-k of v = theta - x_hat
            assert np.array_equal(tko.topk_decode(code[i], n_pad, np.float64, k)[1], tko.topk_select(v[i], live, k))
        theta, s = _np(opt.arena.theta), _np(opt.s)
        x_hat = x_hat + _dec(code, n_pad, k)
        assert np.array_equal(_np(opt.x_hat), x_hat), f"round {r}"


@pytest.mark.parametrize("graph", sorted(STATIC))
def test_beer_torch_path_matches_float64_oracle_round_by_round(graph):
    pr = LeastSquares(STATIC[graph], seed=1)
    opt = BEER(pr, "cpu", _conf("beer"))
    W = metropolis(STATIC[graph][0])
    nbrs = _nbrs(W)
    n_pad, k = opt.arena.n_pad, opt.topk_k
    u = 2.0 ** -53
    for r in range(8):
        st = {n: _np(getattr(opt, n)) for n in ("h", "s_h", "v", "g", "s_g", "m_old")}
        theta = _np(opt.arena.theta)
        dh, dg = _dec(opt.code_h.numpy(), n_pad, k), _dec(opt.code_g.numpy(), n_pad, k)
        opt.run_rounds(1)
        th, sh, sg, e_th, e_sh, e_sg = bo.mix(theta, st["h"], st["s_h"], st["v"], st["s_g"], dh, dg, nbrs, W, 0.5,
                                              0.05, u, 0.0)
        grad = np.zeros_like(th)
        grad[:, :5] = np.stack([pr.grad(i, th[i, :5]) for i in range(pr.N)])
        v, e_v = bo.step_tracker(st["v"], st["g"], sg, st["m_old"], grad, 0.0, 0.5, u)
        for name, got, want in (("theta", _np(opt.arena.theta), th), ("s_h", _np(opt.s_h), sh),
                                ("s_g", _np(opt.s_g), sg), ("v", _np(opt.v), v)):
            np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-12, err_msg=f"round {r} {name}")
        assert np.array_equal(_np(opt.h), st["h"] + _dec(opt.code_h.numpy(), n_pad, k)), f"round {r} h"
        assert np.array_equal(_np(opt.g), st["g"] + _dec(opt.code_g.numpy(), n_pad, k)), f"round {r} g"


@pytest.mark.parametrize("graph", ["random", "wheel", "isolated"])
def test_beer_invariants_hold_every_round(graph):
    """As with the dense codes: s_h + W dec(qh) == W h, s_g + W dec(qg) == W g, sum v == sum m_old and sum theta
    moves by -alpha sum v."""
    g = STATIC[graph][0]
    pr = LeastSquares([g], seed=4)
    opt = BEER(pr, "cpu", _conf("beer", outer_iterations=100))
    W = torch.as_tensor(metropolis(g))
    n_pad, k = opt.arena.n_pad, opt.topk_k
    worst = dict(s=0.0, v=0.0, theta=0.0)
    for _ in range(100):
        sum0, vsum0 = opt.arena.theta.sum(0).clone(), opt.v.sum(0).clone()
        opt.run_rounds(1)
        for s, est, code in ((opt.s_h, opt.h, opt.code_h), (opt.s_g, opt.g, opt.code_g)):
            got = s + W @ ref.choco_decode(code, "topk", n_pad, torch.float64, opt.live, k)
            worst["s"] = max(worst["s"], (got - W @ est).abs().max().item() / max(est.abs().max().item(), 1e-300))
        worst["v"] = max(worst["v"], (opt.v.sum(0) - opt.m_old.sum(0)).abs().max().item()
                         / max(opt.m_old.abs().max().item(), 1e-300))
        moved = opt.arena.theta.sum(0) - sum0
        worst["theta"] = max(worst["theta"], (moved + 0.05 * vsum0).abs().max().item()
                             / max(opt.arena.theta.abs().max().item(), 1e-300))
    print(f"\n{graph} topk: {worst}")
    assert worst["s"] < 1e-13 and worst["v"] < 1e-12 and worst["theta"] < 1e-12


def _rel_to_solution(opt, pr):
    x = pr.solution()
    return np.abs(_np(opt.arena.theta)[:, :len(x)] - x).max() / np.abs(x).max()


def test_topk_beer_is_exact_on_heterogeneous_least_squares():
    """Full gradients, heterogeneous local minimisers, a 10-node cycle, 20 parameters and k = 5: BEER reaches the
    global least-squares solution at every node; CHOCO-SGD with the same codes and DSGD keep the heterogeneity bias."""
    g = [nx.cycle_graph(10)]
    R, alpha, gamma = 3000, 0.05, 0.5
    pr = LeastSquares(g, n=20, m=40, seed=6)
    b = BEER(pr, "cpu", _conf("beer", alpha=alpha, gamma=gamma, topk_ratio=0.25, outer_iterations=R))
    assert b.topk_k == 5
    b.run_rounds(R)
    rb = _rel_to_solution(b, pr)
    pc = LeastSquares(g, n=20, m=40, seed=6)
    c = ChocoSGD(pc, "cpu", _conf("choco_sgd", alpha0=alpha, mu=0.0, gamma=gamma, topk_ratio=0.25, outer_iterations=R))
    c.run_rounds(R)
    rc = _rel_to_solution(c, pc)
    pd = LeastSquares(g, n=20, m=40, seed=6)
    d = DSGD(pd, "cpu", {"alg_name": "dsgd", "alpha0": alpha, "mu": 0.0, "outer_iterations": R})
    d.run_rounds(R)
    rd = _rel_to_solution(d, pd)
    print(f"\ntopk 25 %, {R} rounds: max relative distance to the solution: BEER {rb:.1e}, CHOCO {rc:.1e}, DSGD {rd:.1e}")
    assert rb < 1e-9
    assert rc > 1e-2 and rd > 1e-2


def test_topk_choco_reaches_consensus_on_a_homogeneous_problem():
    """Every node holds the same least-squares problem: CHOCO-SGD with top-k codes (k = 5 of 20) drives the nodes to
    consensus at the common minimiser from different starting rows."""
    g = [nx.cycle_graph(8)]
    pr = LeastSquares(g, n=20, m=40, seed=2)
    pr.A[:] = pr.A[0]
    pr.b[:] = pr.b[0]
    pr._A, pr._b = torch.as_tensor(pr.A), torch.as_tensor(pr.b)
    c = ChocoSGD(pr, "cpu", _conf("choco_sgd", alpha0=0.05, mu=0.0, gamma=0.5, topk_ratio=0.25, outer_iterations=3000))
    th0 = _np(c.arena.theta)[:, :20]
    c.run_rounds(3000)
    th = _np(c.arena.theta)[:, :20]
    spread0 = np.abs(th0 - th0.mean(0)).max()
    spread = np.abs(th - th.mean(0)).max()
    dist = _rel_to_solution(c, pr)
    print(f"\nconsensus spread {spread0:.2e} -> {spread:.2e}, distance to the minimiser {dist:.1e}")
    assert spread < 1e-9 * spread0 and dist < 1e-9


@pytest.mark.parametrize("alg", ["choco_sgd", "beer"])
def test_ratio_one_is_bitwise_none(alg):
    """topk_ratio 1 selects every live element with its exact value: the run is bitwise the compressor none."""
    runs = []
    for comp in ("topk", "none"):
        pr = LeastSquares(STATIC["wheel"], seed=3)
        kw = {"compressor": comp, "topk_ratio": 1.0} if comp == "topk" else {"compressor": "none"}
        conf = _conf(alg, **kw)
        if comp == "none":
            conf.pop("topk_ratio")
        cls = ChocoSGD if alg == "choco_sgd" else BEER
        o = cls(pr, "cpu", conf)
        o.run_rounds(40)
        runs.append([o.arena.theta.clone()] + [getattr(o, n).clone() for n in o.STATE if not n.startswith("code")])
    for x, y in zip(*runs):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ config ----
@pytest.mark.parametrize("alg", ["choco_sgd", "beer"])
def test_config_defaults_and_refusals(alg):
    base = _conf(alg)
    base.pop("topk_ratio")
    c = validate_optimizer(dict(base))
    assert c["topk_ratio"] == ref.TOPK_RATIO_DEFAULT == 0.01
    assert validate_optimizer(dict(base, topk_ratio=1))["topk_ratio"] == 1
    for bad in (0, 0.0, -0.5, 1.5, "0.1", True):
        with pytest.raises(ConfigError, match="topk_ratio"):
            validate_optimizer(dict(base, topk_ratio=bad))
    for comp in ("none", "int8", "sign"):
        with pytest.raises(ConfigError, match="topk_ratio"):
            validate_optimizer(dict(base, compressor=comp, topk_ratio=0.1))
        assert "topk_ratio" not in validate_optimizer(dict(base, compressor=comp))
    pr = LeastSquares(STATIC["cycle"])
    cls = ChocoSGD if alg == "choco_sgd" else BEER
    assert cls(pr, "cpu", dict(base)).topk_k == 1                  # the default ratio: ceil(0.01 * 5)
    with pytest.raises(ValueError, match="topk_ratio"):
        cls(LeastSquares(STATIC["cycle"]), "cpu", dict(base, compressor="int8", topk_ratio=0.5))
    with pytest.raises(ValueError, match="topk_ratio"):
        cls(LeastSquares(STATIC["cycle"]), "cpu", dict(base, topk_ratio=2.0))


def test_compressor_list_is_declared_once():
    from nn_distributed_training_b200.utils import config
    assert config.CHOCO_COMPRESSORS is ref.CHOCO_COMPRESSORS
    assert set(ref.CHOCO_CODE) == set(ref.CHOCO_COMPRESSORS) and ref.CHOCO_CODE["topk"] == 3


def test_topk_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_topk.yaml"), "mnist")
    opts = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [o["alg_name"] for o in opts] == ["dsgt", "choco_sgd", "beer", "beer"]
    assert [o.get("compressor") for o in opts[1:]] == ["topk", "int8", "topk"]
    assert opts[1]["topk_ratio"] == opts[3]["topk_ratio"] == 0.01
    beer = load_experiment(os.path.join(EXP, "dist_mnist_beer.yaml"), "mnist")
    for key in ("graph", "model", "data_split_type", "data_source"):
        assert conf["experiment"].get(key) == beer["experiment"].get(key)
    for p, q in zip(conf["problem_configs"].values(), beer["problem_configs"].values()):
        assert p["train_batch_size"] == q["train_batch_size"]
        assert p["optimizer_config"]["outer_iterations"] == q["optimizer_config"]["outer_iterations"] == 2000


@pytest.mark.parametrize("alg", ["choco_sgd", "beer"])
def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch, alg):
    from test_exact_diffusion import _synthetic
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name=alg)
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = _conf(alg, topk_ratio=0.05, outer_iterations=5)
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    assert {"graph.gpickle", f"{alg}_results.pt"} <= set(os.listdir(outs[0]))
    res = torch.load(os.path.join(outs[0], f"{alg}_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"}
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("alg", ["choco_sgd", "beer"])
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, alg):
    from test_exact_diffusion import _mnist_problem
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    cls = ChocoSGD if alg == "choco_sgd" else BEER
    conf = _conf(alg, topk_ratio=0.02, outer_iterations=6)
    if alg == "beer":
        conf["alpha"] = 0.02
    full = _mnist_problem(conf, N=4, M=100)
    of = cls(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf, N=4, M=100)
    o1 = cls(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf, N=4, M=100)
    o2 = cls(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and all(torch.equal(getattr(o2, n), getattr(o1, n)) for n in cls.STATE)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for n in cls.STATE:
        assert torch.equal(getattr(o2, n), getattr(of, n)), n
    assert second.forward_cnt == full.forward_cnt
