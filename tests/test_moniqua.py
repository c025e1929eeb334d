"""Moniqua on the PyTorch path (CPU, float64): the code layout at every bit width, the decode guarantee and its margin,
unbiasedness, the edge gap, the rounding stream's known answers, the float64 oracle round by round on six graph kinds,
a graph that changes every round and link drops for both bases, invariants 1 to 3 of the mix, the bias Exact
Diffusion's base removes, every configuration refusal, both YAMLs, the runners and checkpoint/resume."""
import copy
import glob
import math
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import moniqua_oracle as mo
from test_exact_diffusion import _mnist_problem, _synthetic
from test_gt_hsgd import GRAPHS, LSProblem
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, Moniqua
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
DROPS = {"link_drop_prob": 0.3, "seed": 5, "from_round": 2, "to_round": 12}
EVERY_ROUND = {"link_drop_prob": 0.4, "seed": 11, "from_round": 0, "to_round": 10 ** 9}
BASE = {"alg_name": "moniqua", "alpha0": 0.05, "bits": 4, "theta_bound": 8.0, "outer_iterations": 10}


def _conf(**kw):
    return dict(BASE, **kw)


def _live(n_pad, n_live):
    live = torch.zeros(n_pad, dtype=torch.bool)
    live[:n_live] = True
    return live


# ------------------------------------------------------------------------------------------------ codes ----
@pytest.mark.parametrize("bits", ref.MQ_BITS)
def test_code_layout_and_packing(bits):
    n_pad, L = 256, 1 << bits
    assert ref.mq_code_bytes(n_pad, bits) == n_pad * bits // 8 and ref.mq_code_bytes(28544, bits) == 28544 * bits // 8
    g = torch.Generator().manual_seed(bits)
    c = torch.randint(0, L, (3, n_pad), generator=g)
    rows = ref.mq_pack(c, bits)
    assert rows.dtype == torch.uint8 and rows.shape == (3, n_pad * bits // 8)
    assert torch.equal(ref.mq_unpack(rows, bits), c)
    words = rows.numpy().view(np.uint32)                  # little-end first: element e at bit (e b) % 32
    for e in (0, 1, 7, 31, 100, n_pad - 1):
        assert (int(words[1, e * bits // 32]) >> (e * bits % 32)) & (L - 1) == int(c[1, e])
    assert np.array_equal(rows[2].numpy(), mo.pack(c[2].numpy(), bits))
    with pytest.raises(ValueError, match="multiple of 128"):
        ref.mq_code_bytes(n_pad + 32, bits)


def test_code_bytes_of_the_paper_mnist_row():
    assert [ref.mq_code_bytes(28544, b) for b in ref.MQ_BITS] == [7136, 14272, 28544]


@pytest.mark.parametrize("bits", ref.MQ_BITS)
def test_decode_guarantee_and_the_same_bits_at_every_reader(bits):
    tb = 0.7
    B, d = ref.mq_range(tb, bits), 2.0 ** -bits
    assert B == pytest.approx(2 * tb / (1 - 2 * d), rel=1e-15)
    n = 4096
    rng = np.random.default_rng(bits)
    x = torch.as_tensor(rng.standard_normal(n) * 50.0)
    live = torch.ones(n, dtype=torch.bool)
    c = ref.mq_codes(x[None], B, bits, torch.as_tensor(rng.random(n))[None], live)[0]
    first = None
    for s in range(40):                                   # readers anywhere within the bound
        y = x + torch.as_tensor(rng.uniform(-tb, tb, n))
        xh, off = ref.mq_decode(c, y, B, bits)
        assert ((xh - x).abs() < B * d).all()
        if first is None:
            first = xh.clone()
        assert torch.equal(xh, first), f"reader {s}"
        xo, _ = mo.decode(c.numpy(), y.numpy(), B, bits)
        assert np.array_equal(xo, xh.numpy())
    own, _ = ref.mq_decode(c, x, B, bits)                 # the node itself decodes the same value
    assert torch.equal(own, first)


@pytest.mark.parametrize("bits", ref.MQ_BITS)
def test_decode_is_unbiased(bits):
    """The mean of xhat - x over many rounding draws is within 5 standard errors of 0 at every element."""
    tb, S = 1.0, 4000
    B = ref.mq_range(tb, bits)
    rng = np.random.default_rng(3)
    x = torch.as_tensor(rng.standard_normal(64) * 10)
    live = torch.ones(64, dtype=torch.bool)
    err = torch.empty(S, 64, dtype=torch.float64)
    key = ref.mq_key(5)
    for s in range(S):
        u = torch.as_tensor(ref.mq_uniforms(key, s, 0, 64))[None]
        xh, _ = ref.mq_decode(ref.mq_codes(x[None], B, bits, u, live)[0], x, B, bits)
        err[s] = xh - x
    se = err.std(0) / math.sqrt(S)
    assert (err.mean(0).abs() < 5 * se + 1e-15).all()
    assert float(err.abs().max()) < B * 2.0 ** -bits


@pytest.mark.parametrize("bits", ref.MQ_BITS)
def test_margin_hits(bits):
    """No hit while |x - y| <= theta_bound - B delta; on data crossing the wrap boundary the oracle counts the hits
    the reference counts, and they are the elements near it."""
    tb = 1.0
    B, d = ref.mq_range(tb, bits), 2.0 ** -bits
    n = 8192
    rng = np.random.default_rng(bits + 10)
    x = torch.as_tensor(rng.standard_normal(n))
    live = torch.ones(n, dtype=torch.bool)
    c = ref.mq_codes(x[None], B, bits, torch.as_tensor(rng.random(n))[None], live)[0]
    y = x + torch.as_tensor(rng.uniform(-1, 1, n)) * (tb - B * d)
    _, off = ref.mq_decode(c, y, B, bits)
    assert not ref.mq_margin_hits(off, bits).any()
    y = x + torch.as_tensor(rng.uniform(-1, 1, n)) * 0.6 * B       # past the bound: some near the wrap
    xh, off = ref.mq_decode(c, y, B, bits)
    hits = ref.mq_margin_hits(off, bits)
    _, ooff = mo.decode(c.numpy(), y.numpy(), B, bits)
    assert int(hits.sum()) == int((np.abs(ooff) > 0.5 - d).sum()) > 0
    wrong = (xh - x).abs() > B * d
    assert wrong.any() and (~hits & ~wrong).any()


def test_edge_gap_ratio():
    rng = np.random.default_rng(0)
    th = torch.as_tensor(rng.standard_normal((6, 50)))
    g = nx.cycle_graph(6)
    want = max(float((th[i] - th[j]).abs().max()) for i, j in g.edges()) / 0.25
    assert ref.mq_edge_gap(th, g.edges(), 0.25) == want
    assert ref.mq_edge_gap(th, [], 0.25) == 0.0


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
], ids=["zeros", "pi"])
def test_rounding_stream_is_philox_with_the_random123_known_answers(ctr, key, want):
    assert [int(x) for x in ref.philox4x32_10(np.array([ctr], dtype=np.uint64), key)[0]] == list(want)
    # the uniforms of elements 4p .. 4p+3 are the four output words of counter (p, k, node, MQ_TAG), times 2^-32
    u = ref.mq_uniforms(key, 7, 3, 16)
    raw = ref.philox4x32_10(np.array([[q, 7, 3, ref.MQ_TAG] for q in range(4)], dtype=np.uint64), key)
    assert np.array_equal(u, raw.reshape(-1).astype(np.float64) * 2.0 ** -32)
    assert ref.mq_key(-1) == (0xFFFFFFFF, 0xFFFFFFFF ^ ref.MQ_KEY_DOMAIN)


# ------------------------------------------------------------------------------------------------ mix ----
MIX_GRAPHS = {"cycle": nx.cycle_graph(8), "star": nx.star_graph(6), "complete": nx.complete_graph(5),
              "path": nx.path_graph(5), "wheel": nx.wheel_graph(7)}


@pytest.mark.parametrize("base", ref.MQ_BASES)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("bits", ref.MQ_BITS)
@pytest.mark.parametrize("graph", sorted(MIX_GRAPHS))
def test_mix_invariants(graph, bits, dtype, base):
    """Invariant 1: the mix conserves the network sum to round-off while every edge is within the bound; 2: each row
    is within 2 (1 - w_ii) B delta of the exact mix of the same rows; 3: padding encodes to 0 and stays 0.  The mix
    equals the oracle launch within its bound, with equal margin counts (zero)."""
    from hsgd_oracle import metropolis
    G = MIX_GRAPHS[graph]
    N, n_pad, n_live, tb = G.number_of_nodes(), 256, 200, 0.5
    W = metropolis(G)
    if base == "exact_diffusion":
        W = ref.ed_weights(W)
    B, d = ref.mq_range(tb, bits), 2.0 ** -bits
    rng = np.random.default_rng(N * bits)
    centre = rng.standard_normal(n_pad) * 30
    th = torch.as_tensor(centre + rng.uniform(-tb / 4, tb / 4, (N, n_pad))).to(dtype)      # edges within tb / 2
    live = _live(n_pad, n_live)
    th[:, ~live] = 0
    codes = ref.mq_unpack(ref.mq_encode(th, B, bits, ref.mq_key(1), 3, range(N), live), bits)
    assert (codes[:, ~live] == 0).all()
    nbrs = [[j for j in G.neighbors(i)] for i in range(N)]
    w_rows = torch.as_tensor(W).to(dtype)
    mixed = th.clone()
    margin = torch.zeros(N, dtype=torch.int64)
    ref.mq_mix_(mixed, codes, w_rows, nbrs, 0, B, bits, margin)
    assert (mixed[:, ~live] == 0).all()
    if bits > 2:                            # tb / 2 <= tb - B delta: no hit (at 2 bits B delta = tb)
        assert (margin == 0).all()
    eps = torch.finfo(dtype).eps
    s0, s1 = th.double().sum(0), mixed.double().sum(0)
    assert ((s1 - s0).abs() <= N * eps * th.double().abs().sum(0) + 1e-12).all()
    exact = w_rows.double() @ th.double()
    lim = 2 * (1 - torch.diagonal(w_rows.double()))[:, None] * B * d
    assert ((mixed.double() - exact).abs() <= lim + 4 * eps * exact.abs() + 1e-12).all()
    want, bound, hits = mo.mix(th.double().numpy(), codes.numpy(), w_rows.double().numpy(), nbrs, 0, B, bits,
                               float(eps))
    assert (np.abs(mixed.double().numpy() - want) <= bound).all() and np.array_equal(hits, margin.numpy())


# ------------------------------------------------------------------------------------------------ oracle ----
CASES = {g: (GRAPHS[g], None) for g in GRAPHS}
CASES["cycle_link_drops"] = (GRAPHS["cycle"], DROPS)
CASES["wheel_every_round"] = (GRAPHS["wheel"], EVERY_ROUND)


@pytest.mark.parametrize("base", ref.MQ_BASES)
@pytest.mark.parametrize("bits", ref.MQ_BITS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_torch_path_matches_float64_oracle_round_by_round(case, bits, base):
    R = 12
    graph, faults = CASES[case]
    pr = LSProblem(graph, batch=8, seed=1, faults=faults)
    graphs = pr.plan_graphs(R, 0, 1)
    if case == "wheel_every_round":
        keys = [tuple(sorted(g.edges())) for g in graphs]
        assert all(a != b for a, b in zip(keys, keys[1:]))
    from hsgd_oracle import metropolis
    Ws = [metropolis(g) for g in graphs]
    # a bound that keeps every decode far from the wrap (|v - n| < 1/3): an ulp of difference cannot change a decode
    opt = Moniqua(pr, "cpu", _conf(bits=bits, base=base, theta_bound=40.0, mu=0.5, outer_iterations=R,
                                   rounding_seed=9))
    live = ref.choco_live(pr.arena.layout).numpy()

    def grad(x, k):
        g = np.zeros_like(x)
        g[:, :5] = pr.batch_grad(x[:, :5], k)
        return g
    want = mo.run(pr.arena.theta.numpy(), Ws, 0.05, 0.5, grad, R, bits, 40.0, ref.mq_key(9), base, live)
    for k, (theta, hits) in enumerate(want):
        opt.run_rounds(1)
        np.testing.assert_allclose(pr.arena.theta.numpy(), theta, rtol=1e-12, atol=1e-12, err_msg=f"round {k}")
        assert np.array_equal(opt.margin.numpy(), hits)
        assert (pr.arena.theta.numpy()[:, 5:] == 0).all()              # invariant 3: the padding stays 0
        codes = ref.mq_unpack(opt.code, bits)
        assert (codes[:, 5:] == 0).all()


def test_exact_diffusion_base_removes_the_heterogeneity_bias():
    """Heterogeneous least squares with full gradients and a constant step: DSGD's fixed point is at least 1e-1 from
    the minimiser.  Moniqua-ED at 8 bits ends at least 5 times closer than DSGD and than Moniqua-DSGD."""
    R, G = 600, nx.cycle_graph(8)
    dist = {}
    for name, conf in [("dsgd", {"alg_name": "dsgd", "alpha0": 0.02, "mu": 0.0, "outer_iterations": R}),
                       ("mq_dsgd", _conf(alpha0=0.02, bits=8, theta_bound=6.0, outer_iterations=R)),
                       ("mq_ed", _conf(alpha0=0.02, bits=8, theta_bound=6.0, base="exact_diffusion",
                                       outer_iterations=R))]:
        pr = LSProblem(G, batch=40, seed=4)
        opt = ALGORITHMS[conf["alg_name"]](pr, "cpu", conf)
        opt.run_rounds(R)
        xs = pr.solution()
        dist[name] = float(np.abs(pr.arena.theta[:, :5].numpy() - xs[None]).max())
        if name != "dsgd":
            assert (opt.margin == 0).all()
    print(f"\nmax distance to the minimiser: {dist}")
    assert dist["dsgd"] >= 1e-1
    assert 5 * dist["mq_ed"] < dist["dsgd"] and 5 * dist["mq_ed"] < dist["mq_dsgd"]


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["moniqua"] is Moniqua
    c = validate_optimizer(dict(BASE))
    assert c["mu"] == 0.0 and c["base"] == "dsgd" and c["update_graph"] is True and "rounding_seed" not in c
    for key in ("consensus_backend", "checkpoint_every", "checkpoint_dir", "resume", "debug_sequence_check"):
        validate_optimizer(dict(BASE, **{key: 1}))
    validate_optimizer(dict(BASE, alpha0=0.0, mu=0.1, bits=2, theta_bound=3, base="exact_diffusion", rounding_seed=-4,
                            update_graph=False, profile=True))
    opt = Moniqua(LSProblem(GRAPHS["cycle"], seed=6), "cpu", _conf())
    assert opt.rounding_seed == 6 and opt.key == ref.mq_key(6) and opt.B == ref.mq_range(8.0, 4)
    assert opt.STATE == ("code", "margin") and opt.psi is None
    assert Moniqua(LSProblem(GRAPHS["cycle"]), "cpu", _conf(base="exact_diffusion")).STATE == ("code", "margin", "psi")


@pytest.mark.parametrize("key", ["alpha0", "bits", "theta_bound", "outer_iterations"])
def test_required_keys(key):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer({k: v for k, v in BASE.items() if k != key})


@pytest.mark.parametrize("key,bad", [
    ("alpha0", -0.1), ("alpha0", float("inf")), ("alpha0", float("nan")), ("alpha0", True),
    ("mu", -0.5), ("mu", float("nan")),
    ("bits", 1), ("bits", 3), ("bits", 16), ("bits", True), ("bits", 4.0), ("bits", "4"),
    ("theta_bound", 0.0), ("theta_bound", -1.0), ("theta_bound", float("inf")), ("theta_bound", False),
    ("base", "dsgt"), ("rounding_seed", 1.5), ("rounding_seed", True)])
def test_out_of_range_values_are_refused(key, bad):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer(dict(BASE, **{key: bad}))
    with pytest.raises(ValueError, match=key):
        Moniqua(LSProblem(GRAPHS["cycle"]), "cpu", _conf(**{key: bad}))


@pytest.mark.parametrize("key", ["gamma", "compressor", "clip_norm", "alpha", "period", "noise_seed"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"moniqua takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        Moniqua(LSProblem(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        Moniqua(LSProblem(GRAPHS["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'moniqua'"):
        validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        Moniqua(LSProblem(nx.cycle_graph(4, create_using=nx.DiGraph)), "cpu", _conf())


# ------------------------------------------------------------------------------------------------ runners ----
MNIST_NAMES = ["dsgd", "exact_diffusion"] + [f"moniqua_{b}_{n}bit" for b in ("dsgd", "ed") for n in (2, 4, 8)]


def test_yamls_validate_and_carry_the_measured_bounds():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_moniqua.yaml"), "mnist")
    pcs = list(conf["problem_configs"].values())
    assert [p["problem_name"] for p in pcs] == MNIST_NAMES
    ocs = [p["optimizer_config"] for p in pcs]
    assert [o["alg_name"] for o in ocs] == ["dsgd", "exact_diffusion"] + ["moniqua"] * 6
    assert [o.get("bits") for o in ocs[2:]] == [2, 4, 8, 2, 4, 8]
    assert [o.get("base") for o in ocs[2:]] == ["dsgd"] * 3 + ["exact_diffusion"] * 3
    hed = load_experiment(os.path.join(EXP, "dist_mnist_hetero_ed.yaml"), "mnist")
    assert conf["experiment"]["graph"] == hed["experiment"]["graph"]
    assert conf["experiment"]["data_split_type"] == "hetero"
    assert all(o["theta_bound"] > 0 for o in ocs[2:])
    dense = load_experiment(os.path.join(EXP, "dist_online_dense_moniqua.yaml"), "online_density")
    names = [p["problem_name"] for p in dense["problem_configs"].values()]
    algs = [p["optimizer_config"]["alg_name"] for p in dense["problem_configs"].values()]
    assert algs[0] == "dsgd" and set(algs[1:]) == {"moniqua"} and len(names) == len(set(names))
    syn = load_experiment(os.path.join(EXP, "dist_online_dense_synthetic.yaml"), "online_density")
    assert dense["experiment"]["data"] == syn["experiment"]["data"]
    for p in dense["problem_configs"].values():
        assert p["dynamic_graph"] is True and p["comm_radius"] == list(syn["problem_configs"].values())[0]["comm_radius"]


def test_mnist_runner_writes_the_moniqua_records(tmp_path, monkeypatch, capsys):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_moniqua.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True, use_cuda=False)
    conf["experiment"]["graph"]["num_nodes"] = 4
    for pc in conf["problem_configs"].values():
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"]["outer_iterations"] = 5
    conf["problem_configs"]["moniqua_dsgd_2bit"]["optimizer_config"]["theta_bound"] = 1e-6    # leaves the guarantee
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_moniqua"))
    assert len(out) == 1
    res = {n: torch.load(os.path.join(out[0], f"{n}_results.pt"), weights_only=False) for n in MNIST_NAMES}
    assert "moniqua_edge_gap" not in res["dsgd"] and "moniqua_margin_hits" not in res["exact_diffusion"]
    for n in MNIST_NAMES[2:]:
        r = res[n]
        assert r["moniqua_margin_hits"].shape == (4,) and r["moniqua_margin_hits"].dtype == torch.int64
        assert len(r["moniqua_edge_gap"]) == 3            # rounds 0, 2 and 4 (the last)
        assert all(torch.isfinite(v).all() for v in r["validation_loss"])
    bad = res["moniqua_dsgd_2bit"]
    assert bad["moniqua_edge_gap"][-1] > 1 and int(bad["moniqua_margin_hits"].sum()) > 0
    assert "moniqua left its decode guarantee" in capsys.readouterr().out
    for n in [n for n in MNIST_NAMES[2:] if not n.endswith("2bit")]:
        assert int(res[n]["moniqua_margin_hits"].sum()) == 0 and max(res[n]["moniqua_edge_gap"]) <= 1


def test_density_runner_runs_moniqua(tmp_path):
    from test_runners import _small_density_conf, _write, synthetic_dir  # noqa: F401
    from nn_distributed_training_b200.experiments import dist_dense_ex
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path / "floor")
    os.makedirs(d)
    write_dataset(d, n_paths=4, seed=0)
    sub = tmp_path / "mq"
    sub.mkdir()
    conf = _small_density_conf("dist_dense_v2.yaml", d, sub)
    conf["experiment"]["graph"] = {"type": "cycle", "num_nodes": 3}
    conf["experiment"]["individual_training"]["train_solo"] = False
    pc = conf["problem_configs"]["problem1"]
    pc.update(train_batch_size=300, val_batch_size=400, problem_name="arm")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "moniqua", "alpha0": 0.01, "bits": 8, "theta_bound": 1.0,
                              "base": "exact_diffusion", "outer_iterations": 4}
    torch.manual_seed(0)
    dist_dense_ex.experiment(_write(str(sub), "d.yaml", conf))
    out = glob.glob(os.path.join(str(sub), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "arm_results.pt"), weights_only=False)
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])
    assert len(res["moniqua_edge_gap"]) == 3 and res["moniqua_margin_hits"].shape == (3,)


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("base", ref.MQ_BASES)
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, base):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(alpha0=0.02, mu=0.5, bits=4, theta_bound=0.5, base=base, outer_iterations=8)
    full = _mnist_problem(conf)
    of = Moniqua(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = Moniqua(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = Moniqua(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and o2.alph == o1.alph and torch.equal(o2.code, o1.code)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta) and torch.equal(o2.code, of.code)
    assert torch.equal(o2.margin, of.margin) and o2.alph == of.alph
    if base == "exact_diffusion":
        assert torch.equal(o2.psi, of.psi)
