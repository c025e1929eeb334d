"""CHOCO-SGD on the PyTorch path (CPU): a float64 oracle round by round, the encoders' properties and byte layout, the
invariants that show every code is applied exactly once, DSGD equivalence, consensus, configuration, the MNIST runner
and checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import choco_oracle as cho
from test_exact_diffusion import GRAPHS, LeastSquares, metropolis
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, DSGD, ChocoSGD
from nn_distributed_training_b200.parallel.arena import FlatLayout, ParamSlot
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
STATIC = {k: v for k, v in GRAPHS.items() if k != "switching"}
COMPRESSORS = ["none", "int8", "sign"]
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
# two slots with an alignment hole and row padding: dead elements inside blocks
LAYOUT = FlatLayout([ParamSlot("a", (5,), 0, 5), ParamSlot("b", (70,), 8, 70), ParamSlot("c", (100,), 80, 100)])


def _conf(comp, **kw):
    return dict({"alg_name": "choco_sgd", "alpha0": 0.05, "mu": 0.0, "gamma": 0.5, "compressor": comp,
                 "outer_iterations": 50}, **kw)


def _v(dtype, L=4, seed=0, layout=LAYOUT):
    g = torch.Generator().manual_seed(seed)
    live = ref.choco_live(layout)
    v = torch.randn(L, layout.n_pad, generator=g, dtype=torch.float64) * torch.exp(
        3 * torch.randn(L, layout.n_pad, generator=g, dtype=torch.float64))
    return (v * live).to(dtype), live


# ------------------------------------------------------------------------------------------------ encoders ----
def test_code_bytes_of_the_paper_model():
    """The published row of the PAPER MNIST model (n_pad = 28 544) in each format."""
    want = {("none", torch.float64): 228352, ("int8", torch.float64): 35680, ("sign", torch.float64): 10704,
            ("none", torch.float32): 114176, ("int8", torch.float32): 32112, ("sign", torch.float32): 7136}
    for (comp, dt), b in want.items():
        assert ref.choco_code_bytes(comp, 28544, dt) == b
        assert b % 16 == 0


@DTYPES
@pytest.mark.parametrize("comp", COMPRESSORS)
def test_byte_layout_round_trip(comp, dtype):
    """encode -> bytes -> decode gives the decoded values encode returned, and the float64 oracle decodes the same
    bytes to the same values (the layout written in tests/choco_oracle.py from csrc/consensus.h)."""
    v, live = _v(dtype)
    codes, dec = ref.choco_encode(v, comp, live)
    assert codes.dtype == torch.uint8 and codes.shape == (4, ref.choco_code_bytes(comp, LAYOUT.n_pad, dtype))
    assert torch.equal(ref.choco_decode(codes, comp, LAYOUT.n_pad, dtype, live), dec)
    npdt = np.float32 if dtype == torch.float32 else np.float64
    for i in range(4):
        d, _ = cho.decode(codes[i].numpy(), comp, LAYOUT.n_pad, npdt, live.numpy())
        np.testing.assert_array_equal(d.astype(npdt), dec[i].numpy())     # int8: the product rounded once
    if comp == "int8":
        q = codes[:, :LAYOUT.n_pad].contiguous().view(torch.int8)
        assert q.abs().max() <= 127 and q.abs().max() == 127
    if comp == "sign":      # bit set exactly where v >= 0
        words = codes[:, :4 * (LAYOUT.n_pad // 32)].contiguous().view(torch.int32).view(-1, LAYOUT.n_pad // 32)
        bits = ((words.to(torch.int64).unsqueeze(-1) >> torch.arange(32)) & 1).reshape(4, -1).bool()
        assert torch.equal(bits, v >= 0)


@DTYPES
@pytest.mark.parametrize("comp", ["int8", "sign"])
def test_contraction_per_block(comp, dtype):
    """||dec(Q(v)) - v||^2 <= (1 - delta) ||v||^2 on every block: delta >= 1 - 32 / 254^2 (int8), and
    delta = ||v||_1^2 / (n_live ||v||^2) (sign, an equality up to rounding)."""
    v, live = _v(dtype, L=8, seed=2)
    _, dec = ref.choco_encode(v, comp, live)
    u = 2.0 ** -24 if dtype == torch.float32 else 2.0 ** -53
    vb, db, lb = v.double().reshape(8, -1, 32), dec.double().reshape(8, -1, 32), live.reshape(-1, 32)
    for i in range(8):
        for b in range(vb.shape[1]):
            x, d, lv = vb[i, b].numpy(), db[i, b].numpy(), lb[b].numpy()
            n2 = (x * x).sum()
            if n2 == 0:
                assert not d.any()
                continue
            e2 = ((d - x) ** 2).sum()
            delta = cho.contraction_delta(x, comp, lv)
            if comp == "int8":
                assert delta >= 1 - 32 / 254 ** 2
            assert e2 <= (1 - delta) * n2 * (1 + 1e-12) + 200 * u * n2, (i, b, e2, n2, delta)


@DTYPES
@pytest.mark.parametrize("comp", COMPRESSORS)
def test_zero_blocks_and_zero_elements(comp, dtype):
    """An all-zero block gets scale 0 and decodes to 0; v = 0 elements of int8 encode to 0; dead elements decode to 0."""
    v, live = _v(dtype)
    v[:, 32:64] = 0
    v[0, 0] = 0
    codes, dec = ref.choco_encode(v, comp, live)
    assert not dec[:, 32:64].any()
    assert not dec[:, ~live].any()
    if comp != "sign":
        assert dec[0, 0] == 0
    if comp == "int8":
        nb = LAYOUT.n_pad // 32
        sc = codes[:, LAYOUT.n_pad:].contiguous().view(dtype).view(-1, nb)
        assert not sc[:, 1].any()


# ------------------------------------------------------------------------------------------------ oracle ----
def _theta(opt):
    return opt.arena.theta.double().numpy().copy()


@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("graph", sorted(STATIC))
def test_torch_path_matches_float64_oracle_round_by_round(graph, comp):
    """The optimizer's rounds against the oracle: the mix from the pending codes, the gradient step; the codes
    themselves are the encoder's (checked above), so the oracle takes x_hat' = x_hat + dec(q) from the published row."""
    pr = LeastSquares(STATIC[graph], seed=1)
    opt = ChocoSGD(pr, "cpu", _conf(comp, mu=0.5))
    W = metropolis(STATIC[graph][0])
    nbrs = [[j for j in range(pr.N) if j != i and W[i, j] != 0] for i in range(pr.N)]
    n_pad, live = opt.arena.n_pad, opt.live.numpy()
    theta, x_hat, s = _theta(opt), np.zeros((pr.N, n_pad)), np.zeros((pr.N, n_pad))
    code = opt.code.numpy().copy()
    alpha, u = 0.05, 2.0 ** -53
    for k in range(8):
        opt.run_rounds(1)
        alpha = alpha * (1.0 - 0.5 * alpha)
        dec = np.stack([cho.decode(code[i], comp, n_pad, np.float64, live)[0] for i in range(pr.N)])
        theta, s, e_th, e_s = cho.mix(theta, x_hat, s, dec, nbrs, W, 0.5, u, 0.0)
        g = np.zeros_like(theta)
        g[:, :5] = np.stack([pr.grad(i, theta[i, :5]) for i in range(pr.N)])
        theta = theta - alpha * g
        np.testing.assert_allclose(_theta(opt), theta, rtol=1e-11, atol=1e-12, err_msg=f"round {k}")
        np.testing.assert_allclose(opt.s.numpy(), s, rtol=1e-11, atol=1e-12, err_msg=f"round {k}")
        code = opt.code.numpy().copy()
        theta = _theta(opt)     # the codes depend on theta to the last bit: continue from the optimizer's state
        s = opt.s.numpy().copy()
        x_hat = x_hat + np.stack([cho.decode(code[i], comp, n_pad, np.float64, live)[0] for i in range(pr.N)])
        np.testing.assert_allclose(opt.x_hat.numpy(), x_hat, rtol=1e-12, atol=1e-13, err_msg=f"round {k}")
        x_hat = opt.x_hat.numpy().copy()
    assert opt.alph == pytest.approx(alpha, rel=1e-15)


def test_isolated_node_takes_plain_sgd_steps():
    """A node without neighbours (W_ii = 1): s equals x_hat after each mix, so theta takes plain SGD steps."""
    pr = LeastSquares(GRAPHS["isolated"], seed=2)
    opt = ChocoSGD(pr, "cpu", _conf("sign"))
    x = _theta(opt)[6, :5]
    for _ in range(5):
        opt.run_rounds(1)
        x = x - 0.05 * pr.grad(6, x)
        dec = ref.choco_decode(opt.code[6:7], "sign", opt.arena.n_pad, torch.float64, opt.live)[0]
        assert torch.equal(opt.s[6] + dec, opt.x_hat[6])
    np.testing.assert_allclose(_theta(opt)[6, :5], x, rtol=1e-13, atol=1e-14)


# ---------------------------------------------------------------------------------------- invariants ----
class Homogeneous(LeastSquares):
    """Every node has the same rows: the minimiser of each node is the global one."""

    def __init__(self, graphs, seed=0, dtype=torch.float64):
        super().__init__(graphs, seed=seed, dtype=dtype)
        self.A[:] = self.A[0]
        self.b[:] = self.b[0]
        self._A = torch.as_tensor(self.A, dtype=dtype)
        self._b = torch.as_tensor(self.b, dtype=dtype)


@pytest.mark.parametrize("comp", COMPRESSORS)
def test_gossip_keeps_the_average_and_s_tracks_x_hat(comp):
    """Over R rounds with a zero gradient: the node average of theta is unchanged by the gossip (to rounding), and
    s_i + sum_j W_ij dec(q_j pending) == sum_j W_ij x_hat_j stays at rounding level."""
    g = GRAPHS["random"][0]
    pr = LeastSquares([g], seed=4)
    opt = ChocoSGD(pr, "cpu", _conf(comp, alpha0=0.0, outer_iterations=200))
    torch.manual_seed(3)
    opt.arena.theta[:, :5] = torch.randn(pr.N, 5, dtype=torch.float64)
    mean0 = opt.arena.theta.mean(0).clone()
    W = torch.as_tensor(metropolis(g))
    worst_mean = worst_s = 0.0
    for _ in range(200):
        opt.run_rounds(1)
        worst_mean = max(worst_mean, (opt.arena.theta.mean(0) - mean0).abs().max().item())
        dec = ref.choco_decode(opt.code, comp, opt.arena.n_pad, torch.float64, opt.live)
        r = (opt.s + W @ dec - W @ opt.x_hat).abs().max().item()
        worst_s = max(worst_s, r / max(opt.x_hat.abs().max().item(), 1e-300))
    spread = (opt.arena.theta - opt.arena.theta.mean(0)).abs().max().item()
    print(f"\n{comp}: |mean drift| {worst_mean:.2e}, |s - W x_hat| / |x_hat| {worst_s:.2e}, spread after 200 "
          f"gossip rounds {spread:.2e}")
    assert worst_mean < 1e-13 and worst_s < 1e-13


@pytest.mark.parametrize("comp", ["int8", "sign"])
def test_compressed_gossip_reaches_consensus_on_a_homogeneous_problem(comp):
    g = [nx.cycle_graph(8)]
    pr = Homogeneous(g, seed=3)
    x_star = pr.solution()
    opt = ChocoSGD(pr, "cpu", _conf(comp, gamma=0.3 if comp == "sign" else 0.8, outer_iterations=4000))
    opt.run_rounds(4000)
    th = _theta(opt)[:, :5]
    spread, err = np.abs(th - th.mean(0)).max(), np.abs(th - x_star).max()
    print(f"\n{comp}: spread {spread:.2e}, |theta - x*|_max {err:.2e}")
    assert spread < 1e-3 and err < 1e-2


@pytest.mark.parametrize("graph", ["cycle", "wheel", "isolated"])
def test_none_with_gamma_one_equals_dsgd(graph):
    """From a common starting row (CHOCO's round 0 has no code to gossip; DSGD's round-0 mix of equal rows is the
    identity), uncompressed CHOCO with gamma = 1 takes DSGD's iterates, up to rounding."""
    pr = LeastSquares(STATIC[graph], seed=5)
    c = ChocoSGD(pr, "cpu", _conf("none", gamma=1.0, mu=0.3, outer_iterations=300))
    c.arena.theta[:] = c.arena.theta[0].clone()
    c.run_rounds(300)
    pr2 = LeastSquares(STATIC[graph], seed=5)
    d = DSGD(pr2, "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.3, "outer_iterations": 300})
    d.arena.theta[:] = d.arena.theta[0].clone()
    d.run_rounds(300)
    r = np.abs(_theta(c) - _theta(d)).max() / np.abs(_theta(d)).max()
    print(f"\nchoco none gamma=1 vs dsgd ({graph}): {r:.2e}")
    assert r < 1e-12


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["choco_sgd"] is ChocoSGD
    base = {"alg_name": "choco_sgd", "alpha0": 0.01, "gamma": 0.5, "compressor": "int8", "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["mu"] == 0.0 and c["update_graph"] is False and c["profile"] is False
    for key in ("alpha0", "gamma", "compressor", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})
    for bad in ({"gamma": 0.0}, {"gamma": 1.5}, {"compressor": "top_k"}, {"mixing_order": "reference"},
                {"update_graph": True}):
        with pytest.raises(ConfigError, match=next(iter(bad))):
            validate_optimizer(dict(base, **bad))
    validate_optimizer(dict(base, gamma=1.0, update_graph=False))
    pr = LeastSquares(GRAPHS["cycle"])
    for bad, msg in (({"mixing_order": "reference"}, "jacobi"), ({"update_graph": True}, "fixed graph"),
                     ({"gamma": 0.0}, "gamma"), ({"compressor": "fp16"}, "compressor")):
        with pytest.raises(ValueError, match=msg):
            ChocoSGD(pr, "cpu", _conf("int8", **bad))


def test_a_changing_graph_is_refused():
    pr = _mnist_problem(_conf("int8"))
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 1}
    with pytest.raises(ValueError, match="fault_injection"):
        ChocoSGD(pr, "cpu", _conf("int8"))
    from nn_distributed_training_b200.optimizers.choco import check_static_plan
    g = nx.cycle_graph(6)
    check_static_plan([g] * 5 + [nx.cycle_graph(6)])       # another object with the same topology
    with pytest.raises(ValueError, match="fixed graph"):
        check_static_plan([g, g, nx.path_graph(6)])


def test_choco_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_choco.yaml"), "mnist")
    opts = [p["optimizer_config"] for p in conf["problem_configs"].values()]
    assert [o["alg_name"] for o in opts] == ["dsgd", "choco_sgd", "choco_sgd"]
    assert [o.get("compressor") for o in opts[1:]] == ["int8", "sign"]
    assert conf["experiment"]["data_split_type"] == "hetero"
    paper = load_experiment(os.path.join(EXP, "dist_mnist_PAPER.yaml"), "mnist")
    for key in ("graph", "model", "data_split_type"):
        assert conf["experiment"][key] == paper["experiment"][key]


# ------------------------------------------------------------------------------------------------ runner ----
def test_mnist_runner_writes_the_reference_layout(tmp_path, monkeypatch):
    from test_exact_diffusion import _synthetic
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="choco_sgd")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "choco_sgd", "alpha0": 0.01, "gamma": 0.5, "compressor": "sign",
                              "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    assert {"graph.gpickle", "choco_sgd_results.pt"} <= set(os.listdir(outs[0]))
    res = torch.load(os.path.join(outs[0], "choco_sgd_results.pt"), weights_only=False)
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
    conf = _conf(comp, alpha0=0.02, mu=0.5, outer_iterations=6)
    full = _mnist_problem(conf)
    of = ChocoSGD(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = ChocoSGD(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = ChocoSGD(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.code, o1.code) and torch.equal(o2.s, o1.s)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for x, y in ((o2.x_hat, of.x_hat), (o2.s, of.s), (o2.code, of.code)):
        assert torch.equal(x, y)
    assert o2.alph == of.alph
    assert second.forward_cnt == full.forward_cnt
