"""GAE(lambda) on the torch paths (rl/gae.py, DistPPOProblem, PPO) against the float64 oracle of ``gae_oracle``, the
``gae_lambda`` refusals and the command-line flags.  The sm_90a scan is held to the same oracle in test_gpu_gae.py."""
import math

import networkx as nx
import numpy as np
import pytest
import torch

from gae_oracle import U, bound, gae64, gae_same_order, normalise64, normalised_bound, rtgs64
from nn_distributed_training_b200.rl import PPO, DistPPOProblem, FFReLUNet, SimpleTagEnv
from nn_distributed_training_b200.rl.gae import check_gae_lambda, gae

DTYPES = {torch.float32: np.float32, torch.float64: np.float64}


def _draw(n, T, E, seed=0):
    g = np.random.default_rng(seed)
    R = n * T * E
    return g.normal(-1.0, 3.0, R), g.normal(0.5, 2.0, R)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_small_case_worked_by_hand(dtype):
    # T = 2, E = 1, gamma = lam = 0.5, r = [1, 2], V = [0.5, 0.25]:
    #   c = 1: delta = 2 - 0.25 = 1.75, A = 1.75, G = 2
    #   c = 0: delta = 1 + 0.5 * 0.25 - 0.5 = 0.625, A = 0.625 + 0.25 * 1.75 = 1.0625, G = 1.5625
    r, v = [1.0, 2.0], [0.5, 0.25]
    A, G = gae(torch.tensor(r, dtype=dtype), torch.tensor(v, dtype=dtype), 0.5, 0.5, 2, 1)
    assert A.tolist() == [1.0625, 1.75] and G.tolist() == [1.5625, 2.0]
    A64, G64 = gae64(r, v, 0.5, 0.5, 2, 1)
    assert A64.tolist() == [1.0625, 1.75] and G64.tolist() == [1.5625, 2.0]


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("gamma", [0.0, 0.95, 0.99, 1.0])
@pytest.mark.parametrize("lam", [0.0, 0.5, 0.95, 1.0])
@pytest.mark.parametrize("n,T,E", [(1, 1, 1), (3, 2, 3), (2, 50, 16), (1, 7, 257)])
def test_torch_scan_is_the_oracle_within_the_bound(n, T, E, lam, gamma, dtype):
    r, v = _draw(n, T, E, seed=T * 1000 + E)
    nd = DTYPES[dtype]
    r, v = r.astype(nd), v.astype(nd)       # the batch-dtype inputs; the oracle sees the same values
    A, G = gae(torch.from_numpy(r), torch.from_numpy(v), gamma, lam, T, E)
    As, Gs = gae_same_order(r, v, gamma, lam, T, E, nd)
    assert np.array_equal(A.numpy(), As) and np.array_equal(G.numpy(), Gs)     # one rounding per op, in order
    A64, G64 = gae64(r, v, gamma, lam, T, E)
    BA, BG = bound(r, v, gamma, lam, T, E, U[nd])
    assert (np.abs(A.numpy() - A64) <= BA).all() and (np.abs(G.numpy() - G64) <= BG).all()


@pytest.mark.parametrize("nd", [np.float32, np.float64])
@pytest.mark.parametrize("gamma", [0.0, 0.9, 0.99, 1.0])
def test_lambda_one_is_rtgs_minus_v_and_lambda_zero_the_td_residual(gamma, nd):
    n, T, E = 3, 50, 4
    r, v = (x.astype(nd) for x in _draw(n, T, E, seed=5))
    u = U[nd]
    rt = rtgs64(r, gamma, T, E)
    A1, G1 = gae_same_order(r, v, gamma, 1.0, T, E, nd)
    BA, BG = bound(r, v, gamma, 1.0, T, E, u)
    assert (np.abs(A1 - (rt - v)) <= BA).all()
    assert (np.abs(G1 - rt) <= BG).all()
    # the float64 oracle itself: A = rtgs - V to float64 round-off
    A64, G64 = gae64(r, v, gamma, 1.0, T, E)
    B64, _ = bound(r, v, gamma, 1.0, T, E, U[np.float64])
    assert (np.abs(A64 - (rt - v)) <= B64).all()
    # lam = 0: delta_c = r_c + gamma V_{c+1} - V_c, V_T = 0
    A0, _ = gae_same_order(r, v, gamma, 0.0, T, E, nd)
    vb = v.reshape(n, T, E).astype(np.float64)
    vn = np.concatenate([vb[:, 1:], np.zeros_like(vb[:, :1])], axis=1)
    td = (r.reshape(n, T, E) + gamma * vn - vb).reshape(-1)
    B0, _ = bound(r, v, gamma, 0.0, T, E, u)
    assert (np.abs(A0 - td) <= B0).all()


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_gamma_zero_and_one_cycle_give_r_minus_v_exactly(dtype):
    r, v = (torch.from_numpy(x).to(dtype) for x in _draw(3, 4, 5, seed=2))
    for lam in (0.0, 0.7, 1.0):
        A, _ = gae(r, v, 0.0, lam, 4, 5)
        assert torch.equal(A, r - v)
    for gamma in (0.5, 1.0):
        A, G = gae(r, v, gamma, 0.9, 1, 5)    # T = 1: every cycle is its own terminal episode
        assert torch.equal(A, r - v) and torch.equal(G, (r - v) + v)


@pytest.mark.parametrize("where", ["reward", "value"])
def test_a_planted_input_does_not_leak_across_episodes_or_worlds(where):
    n, T, E = 3, 6, 4
    r, v = np.zeros(n * T * E), np.zeros(n * T * E)
    blk, c0, e0 = 1, 3, 2
    (r if where == "reward" else v)[(blk * T + c0) * E + e0] = 1.0
    A, _ = gae(torch.from_numpy(r), torch.from_numpy(v), 0.9, 0.8, T, E)
    A = A.numpy().reshape(n, T, E)
    touched = np.zeros_like(A, dtype=bool)
    touched[blk, : c0 + 1, e0] = True
    assert (A[~touched] == 0).all() and (A[touched] != 0).all()
    if where == "reward":
        assert np.allclose(A[blk, : c0 + 1, e0], [(0.9 * 0.8) ** (c0 - c) for c in range(c0 + 1)], rtol=1e-15)


def test_centralized_flattened_layout():
    """PPO's rows are ((ep * T + c) * E + e) * N + i: a scan over T cycles of E * N (world, predator) columns is the
    per-(episode, world, predator) scan."""
    n_ep, T, E, N = 2, 7, 3, 4
    g = np.random.default_rng(3)
    r4, v4 = g.normal(size=(n_ep, T, E, N)), g.normal(size=(n_ep, T, E, N))
    A, G = gae(torch.from_numpy(r4.reshape(-1)), torch.from_numpy(v4.reshape(-1)), 0.99, 0.95, T, E * N)
    ref = np.zeros_like(r4)
    for ep in range(n_ep):
        for e in range(E):
            for i in range(N):
                ref[ep, :, e, i] = gae64(r4[ep, :, e, i], v4[ep, :, e, i], 0.99, 0.95, T, 1)[0]
    BA, _ = bound(r4.reshape(-1), v4.reshape(-1), 0.99, 0.95, T, E * N, U[np.float64])
    assert (np.abs(A.numpy() - ref.reshape(-1)) <= BA).all()


def _env(E=2, dtype=torch.float64):
    return SimpleTagEnv(num_envs=E, num_good=1, num_adversaries=3, num_obstacles=2, max_cycles=200, dtype=dtype, seed=0)


def _dist_problem(lam, dtype=torch.float64, **kw):
    env = _env(dtype=dtype)
    d0 = env.observation_spaces["adversary_0"].shape[0]
    torch.manual_seed(0)
    return DistPPOProblem(FFReLUNet([d0, 16, 5], dtype=dtype), FFReLUNet([d0, 16, 1], dtype=dtype), nx.wheel_graph(3),
                          env, timesteps_per_batch=400, max_timesteps_per_episode=40, gamma=0.95, gae_lambda=lam, **kw)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_dist_ppo_torch_path_against_the_oracle(dtype):
    pr = _dist_problem(0.9, dtype)
    pr.split_rollout_marl()
    T, E, nd = pr._episode_T, pr.env.E, DTYPES[dtype]
    assert T == 10 and len(pr.curr_rews[0]) == len(pr.curr_rtgs[0])
    pr.update_advantage()
    for i in range(pr.N):
        r = pr.curr_rews[i].numpy()
        # the torch rollout's rewards-to-go are the same scan of the same rewards
        assert np.array_equal(pr.curr_rtgs[i].numpy(), gae_same_order(r, np.zeros_like(r), 0.95, 1.0, T, E, nd)[0])
        with torch.no_grad():
            V = pr.models[i].critic(pr.curr_obs[i]).squeeze(-1).numpy()
        A64, G64 = gae64(r, V, 0.95, 0.9, T, E)
        BA, BG = bound(r, V, 0.95, 0.9, T, E, U[nd])
        assert (np.abs(pr.curr_returns[i].numpy() - G64) <= BG).all()
        assert np.array_equal(pr.critic_target(i).numpy(), pr.curr_returns[i].numpy())
        adv = pr.A_k[i].numpy()[None]
        assert (np.abs(adv - normalise64(A64[None])) <= normalised_bound(A64[None], BA[None], U[nd])).all()
    a, c = pr.ev_ppo_loss(0)
    with torch.no_grad():
        V = pr.models[0].critic(pr.curr_obs[0]).squeeze(-1)
    assert torch.equal(c, torch.nn.functional.mse_loss(V, pr.curr_returns[0]))


def test_dist_ppo_without_gae_is_unchanged():
    pr = _dist_problem(None)
    pr.split_rollout_marl()
    pr.update_advantage()
    assert not hasattr(pr, "curr_rews") and not hasattr(pr, "curr_returns")
    for i in range(pr.N):
        with torch.no_grad():
            A = pr.curr_rtgs[i] - pr.models[i].critic(pr.curr_obs[i]).squeeze(-1)
        assert torch.equal(pr.A_k[i], (A - A.mean()) / (A.std() + 1e-10))
        assert pr.critic_target(i) is pr.curr_rtgs[i]


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_centralized_ppo_torch_path_against_the_oracle(dtype):
    env = _env(dtype=dtype)
    m = PPO(FFReLUNet, env, timesteps_per_batch=400, max_timesteps_per_episode=40, gamma=0.99, gae_lambda=0.95,
            seed=0)
    if dtype == torch.float64:
        m.actor.double(); m.critic.double()
    obs, acts, lps, rtgs, _ = m.rollout()
    T, EN, nd = m.episode_T, env.E * env.n_adv, DTYPES[dtype]
    assert T == 10 and m.rews.shape == rtgs.shape
    r = m.rews.numpy()
    assert np.array_equal(rtgs.numpy(), gae_same_order(r, np.zeros_like(r), 0.99, 1.0, T, EN, nd)[0])
    adv, target = m._advantages_torch(obs, acts, rtgs)
    with torch.no_grad():
        V = m.critic(obs).squeeze(-1).numpy()
    A64, G64 = gae64(r, V, 0.99, 0.95, T, EN)
    BA, BG = bound(r, V, 0.99, 0.95, T, EN, U[nd])
    assert (np.abs(target.numpy() - G64) <= BG).all()
    assert (np.abs(adv.numpy()[None] - normalise64(A64[None])) <= normalised_bound(A64[None], BA[None], U[nd])).all()
    m.gae_lambda = None
    adv0, target0 = m._advantages_torch(obs, acts, rtgs)
    assert target0 is rtgs


BAD = [True, False, -0.1, 1.0 + 1e-12, math.nan, math.inf, -math.inf, "0.9", [0.9], 1j]


@pytest.mark.parametrize("value", BAD, ids=repr)
def test_every_gae_lambda_refusal(value):
    with pytest.raises(ValueError, match="gae_lambda"):
        check_gae_lambda(value)
    with pytest.raises(ValueError, match="gae_lambda"):
        _dist_problem(value)
    with pytest.raises(ValueError, match="gae_lambda"):
        PPO(FFReLUNet, _env(), gae_lambda=value)


@pytest.mark.parametrize("value", [None, 0, 0.0, 0.5, 1, 1.0])
def test_accepted_gae_lambdas(value):
    assert check_gae_lambda(value) == (None if value is None else float(value))
    assert _dist_problem(value).gae_lambda == check_gae_lambda(value)


def test_cli_flags_reach_the_problems(monkeypatch):
    from nn_distributed_training_b200.rl import arguments, main as rl_main
    from nn_distributed_training_b200.rl.train_common import make_problem, parse_args

    assert make_problem(parse_args(["--num_envs", "2"]))[0].gae_lambda is None
    pr, hyper = make_problem(parse_args(["--num_envs", "2", "--gae_lambda", "0.95"]))
    assert pr.gae_lambda == 0.95 and hyper["gae_lambda"] == 0.95
    with pytest.raises(ValueError, match="gae_lambda"):
        make_problem(parse_args(["--num_envs", "2", "--gae_lambda", "1.5"]))
    assert arguments.get_args([]).gae_lambda is None
    seen = {}
    monkeypatch.setattr(rl_main, "train", lambda env, hyper, *a: seen.update(hyper))
    rl_main.main(["--num_envs", "2", "--gae_lambda", "0.3"])
    assert seen["gae_lambda"] == 0.3
    model = PPO(FFReLUNet, _env(), **{k: v for k, v in seen.items() if k in PPO.DEFAULTS})
    assert model.gae_lambda == 0.3
