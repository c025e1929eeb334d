"""The fused predator-prey rollout kernel (ops/csrc/tag_rollout.cu) against the float64 replay oracle, its noise, and
the RL entry points that run it.  The yardsticks (``check_fp64``, ``fp32_ratio``) are those of tests/tag_rollout_oracle.py.
"""
import os

import networkx as nx
import numpy as np
import pytest
import torch

from nn_distributed_training_b200.ops import tag_rollout
from nn_distributed_training_b200.rl import DSGDPPO, DSGTPPO, DiNNOPPO, PPO, DistPPOProblem, FFReLUNet, SimpleTagEnv
from nn_distributed_training_b200.rl.eval_policy import load_distributed_actors, rollout as eval_rollout
from tag_rollout_oracle import COV, GAMMA, check_fp64 as _check_fp64, fp32_ratio as _fp32_ratio, on as _on, \
    run_kernel as _run_kernel, tag_env as _env

pytestmark = pytest.mark.gpu
DEV = "cuda"
TRAINED = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nn_distributed_training_b200", "rl",
                       "trained")


def _actors(env, dtype, hidden=(64, 64, 64), seed=1, shipped=False):
    torch.manual_seed(seed)
    if shipped:
        acts = load_distributed_actors(os.path.join(TRAINED, "ppo_actors_tag_dinno_0_3000.pth"),
                                       lambda: FFReLUNet([12, 64, 64, 64, 5]), 3)
        return [a.to(dtype) for a in acts]
    d0 = env.observation_spaces["adversary_0"].shape[0]
    return [FFReLUNet([d0, *hidden, 5], dtype=dtype) for _ in range(env.n_adv)]


def test_fp64_kernel_matches_replay_oracle_distinct_actors():
    cfg = dict(E=16, n_obst=8, max_cycles=200)
    _check_fp64(cfg, _on(_actors(_env(**cfg), torch.float64), DEV), n_ep=2, T=50)


def test_fp64_kernel_matches_replay_oracle_shipped_actors():
    """The trained DiNNO predators keep catching the prey, so contacts are exercised."""
    cfg = dict(E=16, n_obst=8, max_cycles=200)
    out, _ = _check_fp64(cfg, _on(_actors(None, torch.float64, shipped=True), DEV), n_ep=2, T=50)
    assert out["ep_returns"].mean().item() > 0


@pytest.mark.parametrize("cfg,hidden,T", [
    (dict(E=16, n_adv=2, n_obst=0), (64, 64, 64), 50),
    (dict(E=16, n_adv=4, n_good=2, n_obst=2), (16, 16), 50),
    (dict(E=9, n_adv=3, n_good=2, n_obst=8, max_cycles=20), (32, 64, 32, 16), 20),   # max_cycles < cycles: early done
])
def test_fp64_kernel_other_sizes(cfg, hidden, T):
    env = _env(**cfg)
    _check_fp64(cfg, _on(_actors(env, torch.float64, hidden=hidden), DEV), n_ep=2, T=T)


def test_fp64_kernel_many_worlds_per_cta():
    """400 worlds on 132 SMs: 4 worlds per CTA (the 4-world register blocking), and three fp64 actors plus 4 worlds'
    activations exceed the 227 KB of shared memory, so the weights are read in place through L2."""
    cfg = dict(E=200, n_obst=8, max_cycles=200)
    _check_fp64(cfg, _on(_actors(_env(**cfg), torch.float64), DEV), n_ep=2, T=50)


def test_fp32_kernel_many_worlds_per_cta():
    """600 worlds: 4 worlds per CTA with the three fp32 actors staged in shared memory."""
    cfg = dict(E=600, n_obst=8, max_cycles=200)
    _fp32_ratio(cfg, _on(_actors(_env(**cfg), torch.float32), DEV), T=50, n_ep=1)


def test_fp32_kernel_against_fp64_oracle_within_4x_torch_fp32():
    cfg = dict(E=16, n_obst=8, max_cycles=200)
    _fp32_ratio(cfg, _on(_actors(_env(**cfg), torch.float32), DEV), T=50, n_ep=2)
    _fp32_ratio(cfg, _on(_actors(None, torch.float32, shipped=True), DEV), T=50, n_ep=2)


def _cuda_problem(E=16, steps=200, tpb=2000, backend="cuda", device=DEV, hidden=(64, 64, 64), seed=0):
    env = SimpleTagEnv(num_envs=E, num_good=1, num_adversaries=3, num_obstacles=8, max_cycles=steps, device=device, seed=seed)
    torch.manual_seed(seed)
    return DistPPOProblem(FFReLUNet([12, *hidden, 5]), FFReLUNet([12, *hidden, 1]), nx.wheel_graph(3), env,
                          timesteps_per_batch=tpb, max_timesteps_per_episode=steps, gamma=GAMMA, n_updates_per_iteration=2,
                          lr=3e-4, clip=0.2, rollout_backend=backend)


def test_stored_log_probs_are_the_ppo_ratio_denominator():
    pr = _cuda_problem()
    pr.split_rollout_marl()
    n = pr.curr_obs[0].shape[0]
    assert n == 16 * 50 and pr.logger["t_so_far"] == 16 * 50 * 4 and len(pr.logger["batch_rews"]) == 16
    with torch.no_grad():
        for i in range(3):
            _, lp = pr.evaluate(i)
            assert (lp - pr.curr_log_probs[i]).abs().max().item() < 1e-5
    pr.update_advantage()
    for i in range(3):
        a, c = pr.ev_ppo_loss(i)
        assert torch.isfinite(c) and abs(a.item()) < 1e-4


def test_noise_statistics_and_determinism():
    from scipy import stats
    env = _env(E=2048, dtype=torch.float32, max_cycles=50)
    actors = _on(_actors(env, torch.float32, hidden=(16,)), DEV)
    pos0 = tag_rollout.reset_positions(env, 1)
    a = _run_kernel(env, actors, pos0, 50, key=12345, index=3)
    z = a["eps"].double().flatten()
    n = z.numel()
    assert n >= 10 ** 6
    assert abs(z.mean().item()) < 5 / n ** 0.5
    assert abs(z.var().item() - 1) < 5 * (2 / n) ** 0.5
    lag1 = torch.corrcoef(torch.stack([z[:-1], z[1:]]))[0, 1].item()
    assert abs(lag1) < 5 / n ** 0.5
    ks = stats.kstest(z[:200_000].cpu().numpy(), "norm")
    print(f"noise: mean {z.mean().item():.2e} var {z.var().item():.6f} lag-1 {lag1:.2e} KS p {ks.pvalue:.3f}")
    assert ks.pvalue > 1e-3
    b = _run_kernel(env, actors, pos0, 50, key=12345, index=3)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    c = _run_kernel(env, actors, pos0, 50, key=12345, index=4)
    assert (c["eps"] != a["eps"]).float().mean().item() > 0.99
    d = _run_kernel(env, actors, pos0, 50, key=54321, index=3)
    assert (d["eps"] != a["eps"]).float().mean().item() > 0.99


def test_shared_actor_ppo_learns_on_the_kernel(tmp_path):
    env = _env(E=16, dtype=torch.float32, max_cycles=200)
    m = PPO(FFReLUNet, env, timesteps_per_batch=2000, max_timesteps_per_episode=200, n_updates_per_iteration=2, lr=3e-4,
            save_freq=100, out_dir=str(tmp_path), seed=0, rollout_backend="cuda")
    obs, acts, lps, rtgs, lens = m.rollout()
    assert obs.shape == (16 * 50 * 3, 12) and sum(lens) == 16 * 50 * 4
    # [cycle, world, predator] order: predator 0 sees pos_1 - pos_0 where predator 1 sees pos_0 - pos_1
    o = obs.reshape(50, 16, 3, 12)
    assert torch.equal(o[:, :, 0, 4:6], -o[:, :, 1, 4:6])
    torch.testing.assert_close(o[:, :, 0, 2:4] + o[:, :, 0, 4:6], o[:, :, 1, 2:4])
    with torch.no_grad():
        _, cur = m.evaluate(obs, acts)
    assert (cur - lps).abs().max().item() < 1e-5
    m.learn(total_timesteps=3 * 16 * 50 * 4)
    assert len(m.avg_ep_rews) == 3 and all(np.isfinite(m.avg_ep_rews))
    assert all(torch.isfinite(p).all() for p in m.actor.parameters())


def test_deterministic_eval_of_shipped_actors():
    env = _env(E=16, dtype=torch.float32, max_cycles=50, seed=5)
    actors = _on(_actors(None, torch.float32, shipped=True), DEV)
    ret, length, traj = eval_rollout(actors, env, record=True, backend="cuda")
    assert length == 50 and traj.shape == (50, 4, 2) and ret.mean() > 300
    assert np.allclose(traj[-1], env.pos[0].cpu().numpy())
    cfg = dict(E=16, n_obst=8, max_cycles=50, seed=5)
    out, _ = _fp32_ratio(cfg, actors, T=50, n_ep=1, noise=0.0, perturbed_yardstick=True)
    assert out["ep_returns"].mean().item() > 300


@pytest.mark.parametrize("cls,conf", [
    (DiNNOPPO, {"rho_init": 1.0, "rho_scaling": 1.0, "primal_lr_start": 3e-4, "primal_lr_finish": 1e-3,
                "lr_decay_type": "constant", "persistant_primal_opt": False, "primal_iterations": 2}),
    (DSGDPPO, {"alpha0": 3e-4, "mu": 0.0}),
    (DSGTPPO, {"alpha_actor": 3e-4, "alpha_critic": 1e-3}),
])
def test_consensus_trainers_on_the_kernel(tmp_path, cls, conf):
    conf = dict(conf, max_rl_timesteps=3 * 3200, outer_iterations=10 ** 6, ID=4, out_dir=str(tmp_path))
    pr = _cuda_problem(E=16, steps=200, tpb=2000)
    tr = cls(pr, DEV, conf)
    tr.train()
    ref = _cuda_problem(E=16, steps=200, tpb=2000, backend="torch", device="cpu")
    tr_ref = cls(ref, "cpu", dict(conf, out_dir=str(tmp_path / "cpu")))
    tr_ref.train()
    assert tr.timesteps == tr_ref.timesteps == [3200, 6400, 9600]
    assert all(np.isfinite(tr.avg_ep_rews))
    files = set(os.listdir(tmp_path))
    alg = tr.alg
    assert {f"ppo_actors_tag_{alg}_4_0.pth", f"ppo_critics_tag_{alg}_4_0.pth", f"avg_ep_rews_{alg}_4.npy",
            f"timesteps_{alg}_4.npy", f"agreements_{alg}_4.npz"} <= files
