"""SPARQ-SGD on the PyTorch path (CPU): the row and tail layout, the threshold schedule, the float64 oracle round by
round on six graph kinds for every compressor, one to three local steps and three thresholds, the four properties
(s tracks W x_hat, the mix conserves the sum, threshold 0 is CHOCO-SGD bit for bit, a threshold above every error is
local SGD bit for bit), the exact pulled bytes, every configuration refusal, the YAML, the MNIST runner and
checkpoint/resume."""
import copy
import glob
import os

import networkx as nx
import numpy as np
import pytest
import torch
import yaml

import choco_oracle as cho
import sparq_oracle as so
from test_choco import LAYOUT
from test_exact_diffusion import GRAPHS as ED_GRAPHS, LeastSquares, _mnist_problem, _synthetic, metropolis
from test_sgp import _exp
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import ALGORITHMS, ChocoSGD, GossipPGA, SparqSGD
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")
GRAPHS = {k: v for k, v in ED_GRAPHS.items() if k != "switching"}
GRAPHS["star"] = [nx.star_graph(6)]
COMPRESSORS = ["none", "int8", "sign"]
BASE = {"alg_name": "sparq_sgd", "alpha0": 0.05, "mu": 0.5, "gamma": 0.5, "compressor": "int8", "threshold": 0.0,
        "outer_iterations": 50}
# threshold constants c of thr_k = c alpha_k^2: every nonzero difference triggers, some nodes do and some do not
# (None: the median of e_k / alpha_k^2 over a threshold-0 run of the same case), none does
THRESHOLDS = {"zero": 0.0, "mid": None, "never": 1e30}


def _conf(**kw):
    return dict(BASE, **kw)


def _theta(opt):
    return opt.arena.theta.double().numpy().copy()


# ------------------------------------------------------------------------------------------------ layout ----
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("comp", COMPRESSORS)
def test_row_and_tail_layout(comp, dtype):
    """A row is choco_encode's bytes then {uint32 trig, uint32 0, float64 e}; the stride is a multiple of 16."""
    g = torch.Generator().manual_seed(1)
    live = ref.choco_live(LAYOUT)
    v = (torch.randn(3, LAYOUT.n_pad, generator=g, dtype=torch.float64) * live).to(dtype)
    cb = ref.choco_code_bytes(comp, LAYOUT.n_pad, dtype)
    rb = ref.sparq_row_bytes(cb)
    assert rb == cb + 16 == so.row_bytes(cb) and rb % 16 == 0
    rows = torch.zeros(3, rb, dtype=torch.uint8)
    x_hat = torch.zeros_like(v)
    trig, e = ref.sparq_publish_(v.clone(), x_hat, rows, 0.0, comp, live)
    codes, dec = ref.choco_encode(v, comp, live)
    assert trig.all() and torch.equal(rows[:, :cb], codes) and torch.equal(x_hat, dec)
    for i in range(3):
        t, z, ei = so.tail(rows[i].numpy(), cb)
        assert (t, z) == (1, 0) and ei == float(e[i])
        assert ei == pytest.approx(float((v[i].double() ** 2).sum()), rel=1e-15)
    got_t, got_e = ref.sparq_tail_read(rows, cb)
    assert torch.equal(got_t, trig) and torch.equal(got_e, e)
    # a threshold above every error writes the tails {0, e} only
    before = rows.clone()
    trig2, e2 = ref.sparq_publish_(v.clone() * 2, x_hat, rows, 1e300, comp, live)
    assert not trig2.any() and torch.equal(rows[:, :cb], before[:, :cb]) and torch.equal(x_hat, dec)
    assert [so.tail(r.numpy(), cb)[:2] for r in rows] == [(0, 0)] * 3


def test_row_bytes_of_the_paper_model():
    """The PAPER MNIST model (n_pad = 28 544): CHOCO's rows plus 16 bytes."""
    for comp, dt, b in (("int8", torch.float32, 32128), ("sign", torch.float32, 7152), ("none", torch.float64, 228368)):
        assert ref.sparq_row_bytes(ref.choco_code_bytes(comp, 28544, dt)) == b


def test_threshold_schedule():
    alphas = [0.05]
    for _ in range(9):
        alphas.append(ref.dsgd_alpha(alphas[-1], 0.5))
    alphas = alphas[1:]
    for c0, p in ((0.0, 0.0), (3.0, 0.0), (3.0, 0.5), (7.5, 0.9)):
        got = ref.sparq_threshold(c0, p, alphas)
        np.testing.assert_allclose(got, so.threshold(c0, p, alphas), rtol=1e-15, atol=0)
        assert got.dtype == np.float64
    opt = SparqSGD(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(threshold=2.0, threshold_growth=0.5, outer_iterations=9))
    np.testing.assert_array_equal(opt.threshold_table(), ref.sparq_threshold(2.0, 0.5, opt.alpha_table()))
    np.testing.assert_array_equal(opt.threshold_table(4), opt.threshold_table()[:4])


# ------------------------------------------------------------------------------------------------ oracle ----
@pytest.mark.parametrize("H", [1, 2, 3])
@pytest.mark.parametrize("thr", sorted(THRESHOLDS))
@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_torch_path_matches_float64_oracle_round_by_round(graph, comp, thr, H):
    """Each round against the oracle from the optimizer's state before it: the mix over the triggered rows, H exact
    least-squares steps, the error and the trigger decision (equal to the oracle's; no decision lies within a relative
    1e-12 of its threshold), x_hat and the tail."""
    c0 = THRESHOLDS[thr]
    if c0 is None:
        dry = SparqSGD(LeastSquares(GRAPHS[graph], seed=1), "cpu", _conf(compressor=comp, local_steps=H,
                                                                         outer_iterations=8))
        ratios = []
        for a in dry.alpha_table():
            dry.run_rounds(1)
            ratios += (ref.sparq_tail_read(dry.code, dry.code_bytes)[1].numpy() / (a * a)).tolist()
        c0 = float(np.median(ratios))
    pr = LeastSquares(GRAPHS[graph], seed=1)
    opt = SparqSGD(pr, "cpu", _conf(compressor=comp, threshold=c0, local_steps=H, outer_iterations=8))
    W = metropolis(GRAPHS[graph][0])
    nbrs = [[j for j in range(pr.N) if j != i and W[i, j] != 0] for i in range(pr.N)]
    n_pad, live, cb = opt.arena.n_pad, opt.live.numpy(), opt.code_bytes
    thr_tab = opt.threshold_table()
    u = 2.0 ** -53
    decisions = []
    for k in range(8):
        theta, x_hat, s = _theta(opt), opt.x_hat.numpy().copy(), opt.s.numpy().copy()
        rows = opt.code.numpy().copy()
        trig_prev = np.array([so.tail(r, cb)[0] for r in rows], dtype=bool)
        dec = np.stack([cho.decode(r, comp, n_pad, np.float64, live)[0] for r in rows])
        opt.run_rounds(1)
        theta, s, e_th, e_s = so.mix(theta, x_hat, s, dec, trig_prev, nbrs, W, 0.5, u, 0.0)
        np.testing.assert_allclose(opt.s.numpy(), s, rtol=1e-11, atol=1e-12, err_msg=f"round {k}")
        for _ in range(H):
            g = np.zeros_like(theta)
            g[:, :5] = np.stack([pr.grad(i, theta[i, :5]) for i in range(pr.N)])
            theta, _ = so.step(theta, g, 0.0, opt.alpha_table(k + 1)[k], u)
        np.testing.assert_allclose(_theta(opt), theta, rtol=1e-11, atol=1e-12, err_msg=f"round {k}")
        e, _ = so.sqdist(_theta(opt), x_hat, u)
        trig = so.publish(e, thr_tab[k])
        new = opt.code.numpy()
        for i in range(pr.N):
            t, z, ei = so.tail(new[i], cb)
            assert z == 0 and bool(t) == trig[i], f"round {k} node {i}"
            assert ei == pytest.approx(e[i], rel=1e-13, abs=1e-300)
            if thr_tab[k] > 0:
                assert abs(ei - thr_tab[k]) > 1e-12 * thr_tab[k], f"round {k} node {i}: a decision at the threshold"
            want = x_hat[i] + cho.decode(new[i], comp, n_pad, np.float64, live)[0] if t else x_hat[i]
            np.testing.assert_allclose(opt.x_hat.numpy()[i], want, rtol=1e-12, atol=1e-13)
            if not t:
                assert np.array_equal(new[i][:cb], rows[i][:cb]), f"round {k} node {i}: a code body written"
        decisions.append(trig)
    d = np.stack(decisions)
    assert int(opt.triggers.sum()) == int(d.sum()) and np.array_equal(opt.triggers.numpy(), d.sum(0))
    if thr == "zero":
        assert d.all()
    elif thr == "never":
        assert not d.any()
    elif graph != "isolated":
        assert 0 < d.sum() < d.size, "the mid threshold should trigger some node-rounds and not others"


# ---------------------------------------------------------------------------------------- properties ----
def _run_fixed_thr(comp, thr, rounds, alpha0=0.05, graph="random"):
    pr = LeastSquares(GRAPHS[graph], seed=4)
    opt = SparqSGD(pr, "cpu", _conf(compressor=comp, alpha0=alpha0, outer_iterations=rounds))
    opt._thr = np.full(rounds, thr)
    return pr, opt


@pytest.mark.parametrize("comp", COMPRESSORS)
def test_s_tracks_w_x_hat_and_the_mix_conserves_the_sum(comp):
    """Properties 1 and 2 with a fixed threshold that some node-rounds pass and some do not, and no gradient step:
    s_i + sum_j W_ij dec(q_j pending, triggered) == sum_j W_ij x_hat_j, and the node sum of theta is unchanged."""
    pr, opt = _run_fixed_thr(comp, 0.3, 120, alpha0=0.0)
    torch.manual_seed(3)
    opt.arena.theta[:, :5] = torch.randn(pr.N, 5, dtype=torch.float64)
    sum0 = opt.arena.theta.sum(0).clone()
    W = torch.as_tensor(metropolis(GRAPHS["random"][0]))
    worst_s = worst_sum = 0.0
    for _ in range(120):
        opt.run_rounds(1)
        trig, _ = ref.sparq_tail_read(opt.code, opt.code_bytes)
        dec = ref.choco_decode(opt.code[:, :opt.code_bytes], comp, opt.arena.n_pad, torch.float64, opt.live)
        dec = dec * trig[:, None]
        r = (opt.s + W @ dec - W @ opt.x_hat).abs().max().item()
        worst_s = max(worst_s, r / max(opt.x_hat.abs().max().item(), 1e-300))
        worst_sum = max(worst_sum, (opt.arena.theta.sum(0) - sum0).abs().max().item())
    n = int(opt.triggers.sum())
    print(f"\n{comp}: {n} of {120 * pr.N} node-rounds triggered, |s - W x_hat| / |x_hat| {worst_s:.2e}, "
          f"|sum drift| {worst_sum:.2e}")
    assert 0 < n < 120 * pr.N
    assert worst_s < 1e-13 and worst_sum < 1e-12


@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("graph", ["cycle", "wheel", "isolated"])
def test_threshold_zero_with_one_step_is_choco_bit_for_bit(graph, comp):
    """Property 3: every round, theta, x_hat, s and the code bodies of the triggered rows equal CHOCO-SGD's."""
    conf = _conf(compressor=comp, threshold=0.0, outer_iterations=30)
    a, b = LeastSquares(GRAPHS[graph], seed=5), LeastSquares(GRAPHS[graph], seed=5)
    sp = SparqSGD(a, "cpu", copy.deepcopy(conf))
    ch = ChocoSGD(b, "cpu", {k: v for k, v in conf.items() if k != "threshold"} | {"alg_name": "choco_sgd"})
    cb = sp.code_bytes
    for k in range(30):
        sp.run_rounds(1)
        ch.run_rounds(1)
        assert torch.equal(sp.arena.theta, ch.arena.theta), f"round {k}"
        assert torch.equal(sp.x_hat, ch.x_hat) and torch.equal(sp.s, ch.s), f"round {k}"
        trig, _ = ref.sparq_tail_read(sp.code, cb)
        assert torch.equal(sp.code[trig, :cb], ch.code[trig]), f"round {k}"
        assert not ch.code[~trig].view(torch.uint8).any() or comp == "sign"


@pytest.mark.parametrize("comp", COMPRESSORS)
@pytest.mark.parametrize("graph", ["cycle", "complete", "random"])
def test_a_threshold_above_every_error_is_local_sgd_bit_for_bit(graph, comp):
    """Property 4: no node ever triggers, so theta += gamma (0 - 0) and the run is Gossip-PGA's local SGD (``gossip:
    false``, a period past the run) bit for bit; no code body is pulled.  (theta += 0 would turn a -0 into +0; the
    least-squares rows here have no zero element.)"""
    R = 25
    a, b = LeastSquares(GRAPHS[graph], seed=6), LeastSquares(GRAPHS[graph], seed=6)
    sp = SparqSGD(a, "cpu", _conf(compressor=comp, threshold=1e30, outer_iterations=R))
    ls = GossipPGA(b, "cpu", {"alg_name": "gossip_pga", "alpha0": 0.05, "mu": 0.5, "period": R + 1, "gossip": False,
                              "outer_iterations": R})
    sp.run_rounds(R)
    ls.run_rounds(R)
    assert torch.equal(sp.arena.theta, ls.arena.theta)
    assert not sp.triggers.any() and not sp.x_hat.any() and not sp.s.any()
    assert sp.pulled_bytes() == 16 * R * int(sp.pr.topology().deg.sum())


def test_pulled_bytes_count_tails_and_triggered_bodies():
    """pulled = 16 B per neighbor edge and round + code_bytes per trigger of the source that a mix has read."""
    pr, opt = _run_fixed_thr("int8", 0.3, 40, alpha0=0.0)
    torch.manual_seed(3)
    opt.arena.theta[:, :5] = torch.randn(pr.N, 5, dtype=torch.float64)
    deg = np.asarray(opt.pr.topology().deg, dtype=np.int64)
    pulled = 0
    for k in range(40):
        trig_prev, _ = ref.sparq_tail_read(opt.code, opt.code_bytes)
        pulled += 16 * int(deg.sum()) + opt.code_bytes * int((deg * trig_prev.numpy()).sum())
        opt.run_rounds(1)
        assert opt.pulled_bytes() == pulled, f"round {k}"
    assert opt.choco_bytes() == opt.code_bytes * 40 * int(deg.sum())
    assert 0 < opt.pulled_bytes() < opt.choco_bytes()


# ------------------------------------------------------------------------------------------------ config ----
def test_registered_and_config_defaults():
    assert ALGORITHMS["sparq_sgd"] is SparqSGD
    base = {"alg_name": "sparq_sgd", "alpha0": 0.01, "gamma": 0.5, "compressor": "int8", "threshold": 1.0,
            "outer_iterations": 3}
    c = validate_optimizer(dict(base))
    assert c["mu"] == 0.0 and c["local_steps"] == 1 and c["threshold_growth"] == 0.0 and c["update_graph"] is False
    for key in ("alpha0", "gamma", "compressor", "threshold", "outer_iterations"):
        with pytest.raises(ConfigError, match=key):
            validate_optimizer({k: v for k, v in base.items() if k != key})


@pytest.mark.parametrize("key,bad", [
    ("alpha0", -1.0), ("alpha0", float("inf")), ("mu", -0.5), ("gamma", 0.0), ("gamma", 1.5), ("gamma", True),
    ("threshold", -1.0), ("threshold", float("nan")), ("threshold", float("inf")), ("threshold", True),
    ("threshold_growth", -0.1), ("threshold_growth", 1.0), ("local_steps", 0), ("local_steps", 2.0),
    ("local_steps", True), ("compressor", "fp16")])
def test_out_of_range_values_are_refused(key, bad):
    with pytest.raises(ConfigError, match=key):
        validate_optimizer(dict(BASE, **{key: bad}))
    with pytest.raises(ValueError, match=key):
        SparqSGD(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(**{key: bad}))


def test_topk_is_refused():
    with pytest.raises(ConfigError, match="no topk compressor"):
        validate_optimizer(dict(BASE, compressor="topk"))
    with pytest.raises(ValueError, match="topk is not available"):
        SparqSGD(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(compressor="topk"))


@pytest.mark.parametrize("key", ["topk_ratio", "period", "bits", "alpha", "clip_norm", "gossip"])
def test_other_keys_are_refused(key):
    with pytest.raises(ConfigError, match=f"sparq_sgd takes no key '{key}'"):
        validate_optimizer(dict(BASE, **{key: 1}))


def test_update_graph_is_refused():
    with pytest.raises(ConfigError, match="update_graph"):
        validate_optimizer(dict(BASE, update_graph=True))
    with pytest.raises(ValueError, match="fixed graph"):
        SparqSGD(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(update_graph=True))


def test_link_drop_fault_injection_is_refused():
    pr = _mnist_problem(_conf())
    pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 1}
    with pytest.raises(ValueError, match="fault_injection"):
        SparqSGD(pr, "cpu", _conf())


def test_a_planned_sequence_of_more_than_one_topology_is_refused():
    pr = _mnist_problem(_conf())
    opt = SparqSGD(pr, "cpu", _conf(outer_iterations=4))
    g = pr.graph
    pr.plan_graphs = lambda oits, k0, dpr, init=0, refresh=True: [g, g, nx.path_graph(pr.N), g][:oits]
    with pytest.raises(ValueError, match="sparq_sgd needs a fixed graph"):
        opt.run_rounds(1)


@pytest.mark.parametrize("graph_type", ["directed_cycle", "exponential", "random_directed"])
def test_directed_graph_is_refused(graph_type):
    conf = _exp(graph_type)
    conf["problem_configs"]["problem1"]["optimizer_config"] = dict(BASE)
    with pytest.raises(ConfigError, match=r"experiment\.graph.*optimizer_config\.alg_name is 'sparq_sgd'"):
        validate_experiment(conf, "mnist")
    with pytest.raises(ValueError, match="undirected"):
        SparqSGD(LeastSquares([nx.cycle_graph(4, create_using=nx.DiGraph)]), "cpu", _conf())


def test_reference_mixing_order_is_refused():
    with pytest.raises(ConfigError, match="mixing_order"):
        validate_optimizer(dict(BASE, mixing_order="reference"))
    with pytest.raises(ValueError, match="jacobi"):
        SparqSGD(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(mixing_order="reference"))


def test_byzantine_is_refused():
    with pytest.raises(ConfigError, match="byzantine"):
        validate_optimizer(dict(BASE, byzantine={"nodes": [0], "attack": "sign_flip"}))
    with pytest.raises(ValueError, match="Byzantine"):
        SparqSGD(LeastSquares(GRAPHS["cycle"]), "cpu", _conf(byzantine={"nodes": [0], "attack": "sign_flip"}))


# ------------------------------------------------------------------------------------------------ runner ----
NAMES = ["dsgd", "choco_int8", "sparq_int8_low", "sparq_int8_high", "sparq_int8_h2", "sparq_sign"]


def test_sparq_yaml_validates():
    conf = load_experiment(os.path.join(EXP, "dist_mnist_sparq.yaml"), "mnist")
    pcs = list(conf["problem_configs"].values())
    assert [p["problem_name"] for p in pcs] == NAMES
    ocs = [p["optimizer_config"] for p in pcs]
    assert [o["alg_name"] for o in ocs] == ["dsgd", "choco_sgd"] + ["sparq_sgd"] * 4
    assert [o.get("compressor") for o in ocs[1:]] == ["int8"] * 4 + ["sign"]
    assert ocs[2]["threshold"] < ocs[3]["threshold"] and ocs[4]["local_steps"] == 2
    choco = load_experiment(os.path.join(EXP, "dist_mnist_choco.yaml"), "mnist")
    for key in ("graph", "model", "data_split_type"):
        assert conf["experiment"][key] == choco["experiment"][key]


def test_mnist_runner_writes_the_reference_layout_and_the_sparq_records(tmp_path, monkeypatch, capsys):
    dist_mnist_ex = _synthetic(monkeypatch)
    with open(os.path.join(EXP, "dist_mnist_template.yaml")) as f:
        conf = yaml.safe_load(f)
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    conf["experiment"]["graph"]["num_nodes"] = 4
    pc = conf["problem_configs"]["problem1"]
    pc.update(problem_name="sparq_sgd")
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"] = {"alg_name": "sparq_sgd", "alpha0": 0.01, "gamma": 0.5, "compressor": "sign",
                              "threshold": 5000.0, "local_steps": 2, "outer_iterations": 5}
    p = os.path.join(str(tmp_path), "c.yaml")
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    dist_mnist_ex.experiment(p)
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    assert {"graph.gpickle", "sparq_sgd_results.pt"} <= set(os.listdir(outs[0]))
    res = torch.load(os.path.join(outs[0], "sparq_sgd_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch",
                        "sparq_triggers", "sparq_pulled_bytes"}
    assert len(res["validation_loss"]) == 3 and len(res["sparq_pulled_bytes"]) == 3     # rounds 0, 2 and 4
    assert res["sparq_triggers"].shape == (4,) and res["sparq_triggers"].dtype == torch.int64
    pb = res["sparq_pulled_bytes"]
    assert pb[0] == 0 and pb == sorted(pb)
    assert all(torch.isfinite(v).all() for v in res["validation_loss"])
    assert "node-rounds triggered" in capsys.readouterr().out


# ------------------------------------------------------------------------------------------------ resume ----
@pytest.mark.parametrize("comp", COMPRESSORS)
def test_checkpoint_resume_at_an_odd_round_is_bit_exact(tmp_path, comp):
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    conf = _conf(compressor=comp, alpha0=0.02, threshold=20.0, local_steps=2, outer_iterations=8)
    full = _mnist_problem(conf)
    of = SparqSGD(full, "cpu", copy.deepcopy(conf))
    of.train()
    first = _mnist_problem(conf)
    o1 = SparqSGD(first, "cpu", copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = _mnist_problem(conf)
    o2 = SparqSGD(second, "cpu", copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device("cpu")), resume=True)
    assert o2.k == 3 and torch.equal(o2.code, o1.code) and torch.equal(o2.triggers, o1.triggers)
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    for x, y in ((o2.x_hat, of.x_hat), (o2.s, of.s), (o2.code, of.code), (o2.triggers, of.triggers)):
        assert torch.equal(x, y)
    assert o2.alph == of.alph and second.forward_cnt == full.forward_cnt
    print(f"\n{comp}: triggers {of.triggers.tolist()}")
