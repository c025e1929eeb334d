"""GAE(lambda) on sm_90a: the rollout kernel's per-cycle rewards (``rews``), the GAE stage of the advantage pass
(ops/csrc/ppo_update.cu: gae_kernel) and the trainers that run them, against the float64 oracle of ``gae_oracle``.

* ``rews``: the host's rewards-to-go of the kernel's ``rews`` in the batch dtype equal the kernel's ``rtgs`` bit for
  bit, and every other rollout output is the same bits whether ``rews`` is requested or not.
* The GAE stage, from the critic's ``V`` the kernel copies out, equals ``gae_same_order`` (one rounding per op, in
  order) bit for bit in the returns, and is within the oracle's round-off bound of float64; the normalised advantages
  are within ``normalised_bound`` of the float64 normalisation.
"""

import numpy as np
import pytest
import torch

from gae_oracle import U, bound, gae64, gae_same_order, normalise64, normalised_bound
from nn_distributed_training_b200.ops import ppo_update, tag_rollout
from nn_distributed_training_b200.rl import DSGDPPO, DSGTPPO, DiNNOPPO, PPO, FFReLUNet, SimpleTagEnv
from nn_distributed_training_b200.rl.train_common import common_conf, make_problem, parse_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
ND = {torch.float32: np.float32, torch.float64: np.float64}
DT = [torch.float32, torch.float64]


def _env(N, E, dtype, n_obst=2):
    return SimpleTagEnv(num_envs=E, num_good=1, num_adversaries=N, num_obstacles=n_obst, max_cycles=200, device=DEV,
                        dtype=dtype, seed=0)


def _np(t):
    return t.detach().cpu().numpy()


# ---- the rollout kernel's rews ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT, ids=["f32", "f64"])
@pytest.mark.parametrize("N,E,T,n_ep", [(3, 16, 50, 1), (1, 1, 1, 3), (7, 3, 2, 3), (3, 257, 2, 1), (3, 4, 50, 3)])
def test_rollout_rews_give_the_kernel_rtgs_and_change_nothing_else(N, E, T, n_ep, dtype):
    env = _env(N, E, dtype)
    torch.manual_seed(N * 100 + E)
    d0 = env.observation_spaces["adversary_0"].shape[0]
    actor = FFReLUNet([d0, 64, 64, 5], dtype=dtype).to(DEV)
    pos0 = tag_rollout.reset_positions(env, n_ep)
    kw = dict(T=T, n_ep=n_ep, gamma=0.95, cov_var=0.5, key=11, index=3, pos0=pos0)
    plain = tag_rollout.rollout(env, actor, **kw)
    with_r = tag_rollout.rollout(env, actor, rews=True, **kw)
    assert set(with_r) == set(plain) | {"rews"}
    for k in plain:
        assert torch.equal(plain[k], with_r[k]), k
    r = _np(with_r["rews"])
    assert r.shape == (N, n_ep * T * E) and (r == r[:1]).all()            # one shared predator reward
    nd = ND[dtype]
    host = gae_same_order(r.reshape(-1), np.zeros(r.size), 0.95, 1.0, T, E, nd)[0].reshape(r.shape)
    assert np.array_equal(host, _np(with_r["rtgs"]))


# ---- the GAE stage --------------------------------------------------------------------------------------------------
def _critics(N, d0, dtype, seed):
    torch.manual_seed(seed)
    return [FFReLUNet([d0, 64, 64, 1], dtype=dtype).to(DEV) for _ in range(N)]


def _gae_case(N, T, E, n_ep, lam, gamma, dtype, seed=0, d0=12):
    R = n_ep * T * E
    crits = _critics(N, d0, dtype, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    obs = torch.randn(N, R, d0, device=DEV, dtype=dtype, generator=g)
    rews = 3.0 * torch.randn(N, R, device=DEV, dtype=dtype, generator=g) - 1.0
    rtgs = torch.randn(N, R, device=DEV, dtype=dtype, generator=g)
    vals = torch.empty(N, R, device=DEV, dtype=dtype)
    gae = ppo_update.GAE(rews=rews, gamma=gamma, lam=lam, T=T, E=E, values=vals)
    adv, ret = ppo_update.advantages(crits, obs, rtgs, gae=gae)
    return crits, obs, rews, rtgs, vals, adv, ret


def _check_stage(rews, vals, adv, ret, lam, gamma, T, E, dtype):
    nd = ND[dtype]
    r, v = _np(rews), _np(vals)
    A64 = np.empty(r.shape)
    BA = np.empty(r.shape)
    for i in range(r.shape[0]):
        As, Gs = gae_same_order(r[i], v[i], gamma, lam, T, E, nd)
        assert np.array_equal(Gs, _np(ret[i])), ("returns", i)              # bit for bit from the kernel's V
        A64[i], G64 = gae64(r[i], v[i], gamma, lam, T, E)
        BA[i], BG = bound(r[i], v[i], gamma, lam, T, E, U[nd])
        assert (np.abs(As - A64[i]) <= BA[i]).all() and (np.abs(_np(ret[i]) - G64) <= BG).all()
    if r.shape[1] > 1:
        err = np.abs(_np(adv) - normalise64(A64))
        assert (err <= normalised_bound(A64, BA, U[nd])).all(), float(err.max())


@pytest.mark.parametrize("dtype", DT, ids=["f32", "f64"])
@pytest.mark.parametrize("gamma", [0.0, 0.95, 0.99, 1.0])
@pytest.mark.parametrize("lam", [0.0, 0.5, 0.95, 1.0])
def test_gae_stage_against_the_host_and_the_oracle(lam, gamma, dtype):
    T, E, n_ep, N = 50, 16, 3, 3
    _, _, rews, _, vals, adv, ret = _gae_case(N, T, E, n_ep, lam, gamma, dtype)
    _check_stage(rews, vals, adv, ret, lam, gamma, T, E, dtype)


@pytest.mark.parametrize("dtype", DT, ids=["f32", "f64"])
@pytest.mark.parametrize("N", [1, 3, 7])
@pytest.mark.parametrize("n_ep", [1, 3])
@pytest.mark.parametrize("E", [1, 3, 16, 257])
@pytest.mark.parametrize("T", [1, 2, 50])
def test_gae_stage_shapes(T, E, n_ep, N, dtype):
    _, _, rews, _, vals, adv, ret = _gae_case(N, T, E, n_ep, 0.95, 0.99, dtype, seed=T + E + N)
    _check_stage(rews, vals, adv, ret, 0.95, 0.99, T, E, dtype)


def test_gae_values_are_the_critic_and_lambda_one_is_the_plain_pass():
    """fp64: the V the GAE pass copies out is the critic's, and lam = 1 on rewards whose rewards-to-go are the rtgs
    gives the plain pass's advantages."""
    T, E, n_ep, N = 50, 16, 1, 3
    crits, obs, rews, _, vals, adv, ret = _gae_case(N, T, E, n_ep, 1.0, 0.99, torch.float64)
    with torch.no_grad():
        V = torch.stack([c(o).squeeze(-1) for c, o in zip(crits, obs)])
    assert torch.allclose(vals, V, rtol=1e-12, atol=1e-12)
    rt = torch.from_numpy(gae_same_order(_np(rews).reshape(-1), np.zeros(rews.numel()), 0.99, 1.0, T, E,
                                         np.float64)[0].reshape(N, -1)).to(DEV)
    plain = ppo_update.advantages(crits, obs, rt)
    assert torch.allclose(adv, plain, rtol=0, atol=1e-11)
    assert torch.allclose(ret, rt, rtol=0, atol=1e-11)


def test_gae_refusals():
    crits, obs, rews, rtgs, *_ = _gae_case(2, 5, 4, 1, 0.9, 0.9, torch.float32)
    ok = dict(rews=rews, gamma=0.9, lam=0.9, T=5, E=4)
    for bad, what in [(dict(T=3), "divide"), (dict(E=3), "divide"), (dict(T=0), "divide"), (dict(gamma=1.5), "gamma"),
                      (dict(lam=-0.1), "lam"), (dict(lam=float("nan")), "lam"), (dict(rews=rews[:, :-1]), "rews"),
                      (dict(rews=rews.double()), "rews"), (dict(returns=torch.empty(3, device=DEV)), "returns")]:
        with pytest.raises(ValueError, match=what):
            ppo_update.advantages(crits, obs, rtgs, gae=dict(ok, **bad))


def test_gae_is_deterministic_and_writes_the_given_buffers():
    crits, obs, rews, rtgs, vals, adv, ret = _gae_case(3, 50, 257, 1, 0.95, 0.99, torch.float32)
    out, returns = torch.empty_like(adv), torch.empty_like(ret)
    a2, r2 = ppo_update.advantages(crits, obs, rtgs, out=out,
                                   gae=ppo_update.GAE(rews=rews, gamma=0.99, lam=0.95, T=50, E=257, returns=returns))
    assert a2 is out and r2 is returns
    assert torch.equal(a2, adv) and torch.equal(r2, ret)


# ---- the trainers ---------------------------------------------------------------------------------------------------
def test_centralized_layout_on_the_kernels():
    """PPO's flattened batch (rows r * n_adv + i) through the GAE stage with E * n_adv columns: bit for bit the host
    scan, within the oracle's bound, and the cuda update path's advantages agree with the torch path's (fp64)."""
    env = _env(3, 4, torch.float64)
    m = PPO(lambda shape: FFReLUNet(shape, dtype=torch.float64), env, timesteps_per_batch=2000,
            max_timesteps_per_episode=200, gamma=0.99, gae_lambda=0.95, seed=0, rollout_backend="cuda")
    obs, acts, lps, rtgs, _ = m.rollout()
    T, EN = m.episode_T, env.E * env.n_adv
    vals = torch.empty(1, rtgs.numel(), device=DEV, dtype=torch.float64)
    adv, ret = ppo_update.advantages(m.critic, obs[None], rtgs[None],
                                     gae=ppo_update.GAE(rews=m.rews[None], gamma=0.99, lam=0.95, T=T, E=EN, values=vals))
    _check_stage(m.rews[None], vals, adv, ret, 0.95, 0.99, T, EN, torch.float64)
    adv_t, ret_t = m._advantages_torch(obs, acts, rtgs)
    assert torch.allclose(adv[0], adv_t, rtol=0, atol=1e-9) and torch.allclose(ret[0], ret_t, rtol=1e-10, atol=1e-10)


def test_dist_ppo_torch_and_cuda_updates_agree():
    """One fixed batch from the rollout kernel, fp64: advantages, lambda-returns and losses of both update paths."""
    def problem(update):
        args = parse_args(["--num_envs", "4", "--device", DEV, "--rollout", "cuda", "--update", update, "--seed", "0",
                           "--gae_lambda", "0.95"])
        pr, _ = make_problem(args)
        for m in pr.models.values():
            m.double()
        pr.env = _env(3, 4, torch.float64, n_obst=8)
        return pr

    pc, pt = problem("cuda"), problem("torch")
    for i in range(pc.N):
        pt.models[i].load_state_dict(pc.models[i].state_dict())
    pc.split_rollout_marl()
    pt._stack_batch(pc._batch)
    pt._episode_T = pc._episode_T
    pc.update_advantage()
    pt.update_advantage()
    grads = [[torch.empty_like(p) for p in pc.models[i].parameters()] for i in range(pc.N)]
    losses = pc._cuda_grads(grads)
    for i in range(pc.N):
        assert torch.allclose(pc.A_k[i], pt.A_k[i], rtol=0, atol=1e-9)
        assert torch.allclose(pc.curr_returns[i], pt.curr_returns[i], rtol=1e-10, atol=1e-10)
        a, c = pt.ev_ppo_loss(i)
        assert torch.allclose(losses[i], torch.stack([a, c]).detach(), rtol=1e-9, atol=1e-12)


TRAINERS = {
    "dinno": lambda pr, args, h: DiNNOPPO(pr, torch.device(DEV), dict(
        common_conf(args), rho_init=1.0, rho_scaling=1.0, primal_lr_start=h["lr"], primal_lr_finish=0.001,
        lr_decay_type="constant", persistant_primal_opt=False, primal_iterations=h["n_updates_per_iteration"],
        outer_iterations=10_000_000)),
    "dsgd": lambda pr, args, h: DSGDPPO(pr, torch.device(DEV), dict(common_conf(args), alpha0=h["lr"], mu=0.0)),
    "dsgt": lambda pr, args, h: DSGTPPO(pr, torch.device(DEV), dict(common_conf(args), alpha_actor=h["lr"],
                                                                     alpha_critic=h["lr"], init_grads=False)),
}


def _train(name, lam, iters=3):
    args = parse_args(["--num_envs", "16", "--device", DEV, "--rollout", "cuda", "--update", "cuda", "--consensus",
                       "cuda", "--seed", "0", "--no_writeout", "--max_rl_timesteps", str(iters * 3200)]
                      + ([] if lam is None else ["--gae_lambda", str(lam)]))
    pr, hyper = make_problem(args)
    tr = TRAINERS[name](pr, args, hyper)
    tr.train()
    params = torch.cat([torch.nn.utils.parameters_to_vector(m.parameters()) for m in pr.models.values()])
    return tr, pr, params.clone(), list(tr.avg_ep_rews)


@pytest.mark.parametrize("name", sorted(TRAINERS))
def test_trainer_graph_replay_equals_eager(name, monkeypatch):
    runs = []
    for eager in (False, True):
        if eager:
            monkeypatch.setenv("NNDT_NO_GRAPH", "1")
        tr, pr, params, rews = _train(name, 0.95)
        assert tr.inner._program.capturable == (not eager)
        assert pr._returns is pr._bufs["returns"] and pr._batch["rews"] is pr._bufs["rews"]
        assert len(rews) == 3 and torch.isfinite(params).all()
        runs.append((params, rews))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]
    _, _, plain, _ = _train(name, None)
    assert not torch.equal(plain, runs[0][0])      # GAE changed the update
