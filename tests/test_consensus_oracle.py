"""CPU checks of the float64 consensus oracle (``tests/consensus_oracle.py``): it agrees with the PyTorch consensus ops
(``ops/consensus_ref.py``) launch by launch within its own round-off bound, rounds composed from it reproduce the
PyTorch-path optimizers, and the edge cases (isolated node, complete graph, per-round graph switches) behave."""
import math

import networkx as nx
import numpy as np
import pytest
import torch

import consensus_oracle as co
from nn_distributed_training_b200.ops import consensus_ref as ref
from nn_distributed_training_b200.optimizers import DiNNO, DSGD, DSGT
from nn_distributed_training_b200.utils.graph_generation import Topology

C = 16           # roundings on the longest path of a launch
U = co.U64

GRAPHS = {
    "path2": nx.path_graph(2),
    "cycle5": nx.cycle_graph(5),
    "star8": nx.star_graph(8),
    "wheel10": nx.wheel_graph(10),
    "isolated": nx.Graph([(0, 1), (1, 2), (2, 3), (3, 0), (0, 2)]),
    "complete6": nx.complete_graph(6),
}
GRAPHS["isolated"].add_node(4)


def _random_state(N, n, S, seed, near=None):
    """Rows drawn at random, or within ``near`` (relative) of one common row; every array float64."""
    r = np.random.default_rng(seed)
    if near is None:
        theta = r.normal(size=(N, n))
    else:
        theta = r.normal(size=n) * (1.0 + near * r.normal(size=(N, n)))
    st = dict(theta=theta, dual=r.normal(size=(N, n)) * 0.1, delta=r.normal(size=(N, n)),
              m=r.normal(size=(N, n)) * 0.1, v=r.random(size=(N, n)) * 0.01, g_old=r.normal(size=(N, n)),
              grad_part=r.normal(size=(N, S, n)))
    pub = np.zeros((2, 2, N, n))
    pub[0, 0] = theta
    pub[0, 1] = r.normal(size=(N, n))
    st["pub"] = pub
    return st


def _t(x):
    return torch.as_tensor(np.array(x))


@pytest.mark.parametrize("near", [None, 1e-9])
@pytest.mark.parametrize("opt", ["sgd", "adam", "adamw"])
@pytest.mark.parametrize("gname", ["cycle5", "wheel10", "isolated", "complete6"])
def test_dinno_oracle_matches_torch_ops(gname, opt, near):
    """Exchange, dual ascent and three primal steps against consensus_ref.  Near consensus (rows 1e-9 apart) the
    delta bound is 1e-9 of the sum-form's, so an exchange that adds the rows before subtracting fails here."""
    topo = Topology(GRAPHS[gname])
    N, n, pits, k, rho, lr = topo.N, 64, 3, 1, 0.7, 0.01
    st = _random_state(N, n, 1, seed=N + len(opt), near=near)
    st["pub"][1, 0] = st["theta"]         # round 1 reads parity 1
    theta, theta_k = _t(st["theta"]), _t(st["theta"])
    dual, delta = _t(st["dual"]), torch.zeros(N, n, dtype=torch.float64)
    m, v = torch.zeros(N, n, dtype=torch.float64), torch.zeros(N, n, dtype=torch.float64)
    adj, deg = _t(topo.adj.astype(np.float64)), _t(topo.deg.astype(np.float64))
    ref.dinno_exchange_(theta_k, theta, adj, deg, rho, dual, delta)
    o = st
    for step in range(pits):
        o, err = co.dinno_update(o, step=step, k=k, nbrs=topo.neighbors_noself, rho=rho, lr=lr, opt=opt, pits=pits,
                                 persistent=False, u=U, dtype=np.float64)
        g = ref.dinno_grad(theta, theta_k, _t(st["grad_part"][:, 0]), dual, delta, deg, rho)
        ref.optimizer_step_(theta, g, opt, lr, m, v, step + 1)
        if step == 0:
            co.check("delta", delta, o["delta"], err["delta"], C)
            co.check("dual", dual, o["dual"], err["dual"], C)
        co.check(f"theta step {step}", theta, o["theta"], err["theta"], C)
        if opt != "sgd":
            co.check("m", m, o["m"], err["m"], C)
            co.check("v", v, o["v"], err["v"], C)
        # only the last step publishes, into parity 0 for round 1
        assert np.array_equal(o["pub"][0, 0], o["theta"] if step == pits - 1 else st["pub"][0, 0])
        # the next step starts from the torch state, so each comparison covers one launch
        o = dict(o, theta=theta.numpy().copy(), dual=dual.numpy().copy(), delta=delta.numpy().copy(),
                 m=m.numpy().copy(), v=v.numpy().copy())


@pytest.mark.parametrize("near", [None, 1e-9])
@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_mixing_oracles_match_torch_ops(gname, near):
    topo = Topology(GRAPHS[gname])
    N, n, S, k, alpha = topo.N, 48, 5, 0, 0.03
    st = _random_state(N, n, S, seed=7 * N, near=near)
    W = _t(topo.W)
    nb = topo.neighbors_noself
    o, err = co.dsgd_mix(st, k=k, nbrs=nb, W=topo.W, u=U)
    co.check("dsgd_mix", ref.dsgd_mix(_t(st["theta"]), W), o["theta"], err["theta"], C)
    o, err = co.dsgd_step(st, k=k, alpha=alpha, u=U)
    th = _t(st["theta"])
    ref.dsgd_step_(th, _t(st["grad_part"].sum(1)), alpha)
    co.check("dsgd_step", th, o["theta"], err["theta"], C)
    assert np.array_equal(o["pub"][1, 0], o["theta"])
    o, err = co.dsgt_mix(st, k=k, nbrs=nb, W=topo.W, alpha=alpha, u=U)
    co.check("dsgt_mix", ref.dsgt_mix(_t(st["theta"]), _t(st["pub"][0, 1]), W, alpha), o["theta"], err["theta"], C)
    o, err = co.dsgt_track(st, k=k, nbrs=nb, W=topo.W, u=U)
    y = ref.dsgt_track(_t(st["pub"][0, 1]), W, _t(st["grad_part"].sum(1)), _t(st["g_old"]))
    co.check("dsgt_track", y, o["pub"][1, 1], err["pub"][1, 1], C)
    assert np.array_equal(o["pub"][1, 0], st["theta"]) and np.array_equal(o["g_old"], st["grad_part"].sum(1))


@pytest.mark.parametrize("alg", ["dinno", "dsgd", "dsgt"])
def test_sum_mode_oracles_match_pointer_oracles_on_complete_graph(alg):
    """The complete-graph formulas (network sum, S - N theta_i, (S_theta - alpha S_y) / N) are the pointer-table
    update with uniform weights 1/N."""
    topo = Topology(nx.complete_graph(6))
    st = _random_state(6, 32, 2, seed=3)
    sums = co.local_sum(st["pub"], 0)
    kw = dict(k=0, nbrs=topo.neighbors_noself, u=U)
    if alg == "dinno":
        a = co.dinno_update(st, step=0, rho=0.4, lr=0.01, opt="adam", pits=1, persistent=False, dtype=np.float64, **kw)
        b = co.dinno_update(st, step=0, rho=0.4, lr=0.01, opt="adam", pits=1, persistent=False, dtype=np.float64,
                            sum_mode=True, sums=sums, **kw)
        keys = ("delta", "dual", "theta")
    elif alg == "dsgd":
        a, b = co.dsgd_mix(st, W=topo.W, **kw), co.dsgd_mix(st, W=topo.W, sum_mode=True, sums=sums, **kw)
        keys = ("theta",)
    else:
        a = co.dsgt_mix(st, W=topo.W, alpha=0.05, **kw)
        b = co.dsgt_mix(st, W=topo.W, alpha=0.05, sum_mode=True, sums=sums, **kw)
        keys = ("theta",)
    for key in keys:
        co.check(key, b[0][key], a[0][key], a[1][key] + b[1][key], C)


def test_consensus_metric_oracle_matches_torch_ops():
    r = np.random.default_rng(5)
    rows = r.normal(size=(7, 300)) * (1 + 0.1 * np.arange(7))[:, None]
    rows[3] = rows[2] * 2.5                       # same direction: distance 0 after normalisation
    (pair, e_pair), (mean, e_mean) = co.consensus_metric(rows)
    d_all, d_mean = ref.consensus_error(_t(rows))
    co.check("pair", d_all, pair, e_pair, C)
    co.check("mean", d_mean[:, 0], mean, e_mean, C)
    assert pair[2, 3] < 1e-15 and np.all(np.diag(pair) == 0)


# ------------------------------------------------------------------------------------ composed rounds ----
class _LstsqProblem:
    """Reference-API problem with a deterministic least-squares loss 0.5 |X_i w - y_i|^2 per node, so the oracle can
    evaluate the same gradient in closed form.  ``graphs`` (one per round) makes the graph switch every round."""

    def __init__(self, graphs, n_in=6, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.graphs = list(graphs)
        self.graph = self.graphs[0]
        self.N = self.graph.number_of_nodes()
        self.models = [torch.nn.Linear(n_in, 1, bias=False).double() for _ in range(self.N)]
        for mdl in self.models:
            with torch.no_grad():
                mdl.weight.copy_(torch.randn(1, n_in, generator=g, dtype=torch.float64))
        self.X = [torch.randn(9, n_in, generator=g, dtype=torch.float64) for _ in range(self.N)]
        self.Y = [torch.randn(9, generator=g, dtype=torch.float64) for _ in range(self.N)]
        self.conf = {"metrics_config": {"evaluate_frequency": 100}}
        self._r = 0

    def local_batch_loss(self, i):
        return 0.5 * ((self.models[i](self.X[i])[:, 0] - self.Y[i]) ** 2).sum()

    def update_graph(self):
        self.graph = self.graphs[min(self._r, len(self.graphs) - 1)]
        self._r += 1

    def evaluate_metrics(self, at_end=False):
        pass

    def grad_rows(self, theta):
        """[N, n_pad] gradient of every node at the rows ``theta`` (padding stays 0)."""
        g = np.zeros_like(theta)
        n = self.X[0].shape[1]
        for i in range(self.N):
            X, y = self.X[i].numpy(), self.Y[i].numpy()
            g[i, :n] = X.T @ (X @ theta[i, :n] - y)
        return g


SEQ = [nx.cycle_graph(5), GRAPHS["isolated"], nx.complete_graph(5), nx.star_graph(4), nx.path_graph(5)]
DINNO = {"alg_name": "dinno", "rho_init": 0.3, "rho_scaling": 1.1, "outer_iterations": 5, "primal_iterations": 2,
         "primal_optimizer": "adam", "persistant_primal_opt": False, "primal_lr_start": 0.02,
         "primal_lr_finish": 0.002, "lr_decay_type": "log", "profile": False}


@pytest.mark.parametrize("opt,persistent,decay", [("adam", False, "log"), ("adamw", True, "linear"),
                                                  ("sgd", False, "constant"), ("adam", True, "log")])
@pytest.mark.parametrize("switch", [False, True])
def test_composed_dinno_rounds_reproduce_torch_optimizer(opt, persistent, decay, switch):
    graphs = SEQ if switch else [SEQ[1]] * 5
    pr = _LstsqProblem(graphs)
    conf = dict(DINNO, primal_optimizer=opt, persistant_primal_opt=persistent, lr_decay_type=decay)
    o = DiNNO(pr, "cpu", conf)
    st = dict(theta=o.arena.theta.numpy().copy(), dual=np.zeros_like(o.arena.theta.numpy()))
    st.update(delta=np.zeros_like(st["theta"]), m=np.zeros_like(st["theta"]), v=np.zeros_like(st["theta"]))
    pub = np.zeros((2, 1) + st["theta"].shape)
    pub[0, 0] = st["theta"]
    st["pub"] = pub
    oits, pits = conf["outer_iterations"], conf["primal_iterations"]
    rho, lr = co.rho_table(conf, oits), co.lr_table(conf, oits)
    o.run_rounds(oits)
    for k in range(oits):
        topo = Topology(graphs[k])
        for p in range(pits):
            st["grad_part"] = pr.grad_rows(st["theta"])[:, None, :]
            st, _ = co.dinno_update(st, step=p, k=k, nbrs=topo.neighbors_noself, rho=rho[k], lr=lr[k], opt=opt,
                                    pits=pits, persistent=persistent, u=U, dtype=np.float64)
    np.testing.assert_allclose(o.arena.theta.numpy(), st["theta"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(o.duals.numpy(), st["dual"], rtol=1e-10, atol=1e-12)
    assert np.all(st["theta"][:, 6:] == 0)


@pytest.mark.parametrize("switch", [False, True])
@pytest.mark.parametrize("alg,init", [("dsgd", None), ("dsgt", True), ("dsgt", False)])
def test_composed_mixing_rounds_reproduce_torch_optimizers(alg, init, switch):
    graphs = SEQ if switch else [SEQ[0]] * 5
    pr = _LstsqProblem(graphs, seed=1)
    oits = 5
    if alg == "dsgd":
        conf = {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5, "outer_iterations": oits, "profile": False}
        o = DSGD(pr, "cpu", conf)
    else:
        conf = {"alg_name": "dsgt", "alpha": 0.03, "init_grads": init, "outer_iterations": oits, "profile": False}
        o = DSGT(pr, "cpu", conf)
    theta = o.arena.theta.numpy().copy()
    pub = np.zeros((2, 2) + theta.shape)
    pub[0, 0] = theta
    st = dict(theta=theta, pub=pub, g_old=np.zeros_like(theta))
    o.run_rounds(oits)
    if alg == "dsgt" and init:
        st["grad_part"] = pr.grad_rows(st["theta"])[:, None, :]
        st, _ = co.dsgt_init(st, u=U)
    alphas = co.dsgd_alpha_table(0.05, 0.5, oits)
    for k in range(oits):
        topo = Topology(graphs[k])
        kw = dict(k=k, nbrs=topo.neighbors_noself, W=topo.W, u=U)
        if alg == "dsgd":
            st, _ = co.dsgd_mix(st, **kw)
            st["grad_part"] = pr.grad_rows(st["theta"])[:, None, :]
            st, _ = co.dsgd_step(st, k=k, alpha=alphas[k], u=U)
        else:
            st, _ = co.dsgt_mix(st, alpha=0.03, **kw)
            st["grad_part"] = pr.grad_rows(st["theta"])[:, None, :]
            st, _ = co.dsgt_track(st, **kw)
    np.testing.assert_allclose(o.arena.theta.numpy(), st["theta"], rtol=1e-10, atol=1e-12)
    if alg == "dsgt":
        np.testing.assert_allclose(o.y.numpy(), st["pub"][oits & 1, 1], rtol=1e-10, atol=1e-12)


# --------------------------------------------------------------------------------------------- edges ----
def test_isolated_node_has_zero_delta_and_keeps_its_row():
    topo = Topology(GRAPHS["isolated"])
    assert topo.deg[4] == 0 and topo.W[4, 4] == 1.0
    st = _random_state(5, 16, 3, seed=11)
    o, err = co.dinno_update(st, step=0, k=0, nbrs=topo.neighbors_noself, rho=0.5, lr=0.1, opt="sgd", pits=1,
                             persistent=False, u=U, dtype=np.float64)
    assert np.all(o["delta"][4] == 0) and np.all(err["delta"][4] == 0)
    assert np.array_equal(o["dual"][4], st["dual"][4])
    o, _ = co.dsgd_mix(st, k=0, nbrs=topo.neighbors_noself, W=topo.W, u=U)
    assert np.array_equal(o["theta"][4], st["theta"][4])


def test_consensus_is_a_fixed_point_of_every_oracle():
    """All rows equal, zero duals, zero gradient: delta is exactly 0 with a zero bound, DiNNO's fresh Adam step and
    the mixings on a graph with power-of-two Metropolis weights (3-regular: 1/4) return the row exactly."""
    topo = Topology(nx.cubical_graph())
    N, n = topo.N, 32
    row = np.random.default_rng(2).integers(-512, 512, n) / 64.0
    st = dict(theta=np.tile(row, (N, 1)), dual=np.zeros((N, n)), delta=np.zeros((N, n)), m=np.zeros((N, n)),
              v=np.zeros((N, n)), g_old=np.zeros((N, n)), grad_part=np.zeros((N, 2, n)))
    st["pub"] = np.stack([np.stack([st["theta"], np.zeros((N, n))])] * 2)
    o, err = co.dinno_update(st, step=0, k=0, nbrs=topo.neighbors_noself, rho=0.5, lr=0.1, opt="adam", pits=1,
                             persistent=False, u=U, dtype=np.float64)
    assert np.all(o["delta"] == 0) and np.all(err["delta"] == 0) and np.array_equal(o["theta"], st["theta"])
    for f in (co.dsgd_mix, co.dsgt_mix):
        kw = dict(alpha=0.1) if f is co.dsgt_mix else {}
        assert np.array_equal(f(st, k=0, nbrs=topo.neighbors_noself, W=topo.W, u=U, **kw)[0]["theta"], st["theta"])


def test_schedules_match_the_optimizers():
    for decay in ("constant", "linear", "log"):
        for persistent in (False, True):
            conf = dict(DINNO, lr_decay_type=decay, persistant_primal_opt=persistent, outer_iterations=6)
            o = DiNNO(_LstsqProblem([nx.cycle_graph(5)]), "cpu", conf)
            np.testing.assert_allclose([o.lr_at(k) for k in range(6)], co.lr_table(conf, 6), rtol=1e-14)
            np.testing.assert_allclose([o.rho_at(k) for k in range(6)], co.rho_table(conf, 6), rtol=1e-14)
    o = DSGD(_LstsqProblem([nx.cycle_graph(5)]), "cpu", {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.5,
                                                        "outer_iterations": 6, "profile": False})
    np.testing.assert_allclose(o.alpha_table(), co.dsgd_alpha_table(0.05, 0.5, 6), rtol=1e-15)


def test_affine_perturbation_on_a_cycle_gives_exact_interior_delta():
    """theta_l = theta_0 (1 + 0.03 l) on cycle_graph(4): in exact arithmetic delta of nodes 1 and 2 is 0.  With
    differences accumulated per neighbor (theta_0 - theta_1 and theta_2 - theta_1 are exact, and so is their sum) the
    exchange returns the exact delta of the stored rows, a few units of round-off of theta; taking sums first leaves
    a different residue.  On coordinates without a loss gradient Adam turns the sign of that residue into a full
    +-lr step, which is why a whole-run comparison must not start from such rows.  When the rows are exactly affine
    (dyadic values) the interior delta is exactly 0."""
    r = np.random.default_rng(0)
    th0 = r.normal(size=200)
    topo = Topology(nx.cycle_graph(4))
    adj, deg = _t(topo.adj.astype(np.float64)), _t(topo.deg.astype(np.float64))
    for rows, exact_zero in ((np.stack([th0 * (1.0 + 0.03 * l) for l in range(4)]), False),
                             (np.stack([np.round(th0 * 64) / 64 + l / 32.0 for l in range(4)]), True)):
        theta = _t(rows)
        dual, delta = torch.zeros_like(theta), torch.zeros_like(theta)
        ref.dinno_exchange_(theta, theta, adj, deg, 0.5, dual, delta)
        for i in (1, 2):
            exact = [math.fsum([rows[i - 1, c], rows[i + 1, c], -rows[i, c], -rows[i, c]]) for c in range(200)]
            np.testing.assert_array_equal(delta[i].numpy(), exact)
            if exact_zero:
                assert np.all(delta[i].numpy() == 0)
            else:
                assert np.abs(delta[i].numpy()).max() <= 4 * U * np.abs(rows).max()
        o, _ = co.dinno_update(dict(theta=rows, pub=np.stack([rows[None], rows[None]]), dual=np.zeros_like(rows),
                                    delta=np.zeros_like(rows), m=None, v=None, grad_part=np.zeros((4, 1, 200))),
                               step=0, k=0, nbrs=topo.neighbors_noself, rho=0.5, lr=0.1, opt="sgd", pits=1,
                               persistent=False, u=U, dtype=np.float64)
        np.testing.assert_array_equal(o["delta"], delta.numpy())
