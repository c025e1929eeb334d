"""The fused predator-prey rollout kernel (ops/csrc/tag_rollout.cu) against the float64 replay oracle, its noise, and
the RL entry points that run it.

Contacts are stiff, so rounding differences grow along a trajectory.  The fp64 kernel is therefore held to a
yardstick: the oracle's own divergence when ``pos0`` moves by one ulp (running max over the cycles so far, taken over
all worlds); the kernel's error must stay within 10x of it, with a floor of 1e-12 of the quantity's scale.  The fp32
kernel is held to 4x the error of the torch fp32 path against the same fp64 oracle, with a floor of a few fp32 ulps.
"""
import os

import networkx as nx
import numpy as np
import pytest
import torch

from nn_distributed_training_b200.ops import tag_rollout
from nn_distributed_training_b200.rl import DSGDPPO, DSGTPPO, DiNNOPPO, PPO, DistPPOProblem, FFReLUNet, SimpleTagEnv
from nn_distributed_training_b200.rl.eval_policy import load_distributed_actors, rollout as eval_rollout
from tag_rollout_oracle import replay_tag_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda"
TRAINED = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nn_distributed_training_b200", "rl",
                       "trained")
GAMMA, COV = 0.99, 0.5


def _env(E=16, n_adv=3, n_good=1, n_obst=8, max_cycles=200, dtype=torch.float64, device=DEV, seed=0):
    return SimpleTagEnv(num_envs=E, num_good=n_good, num_adversaries=n_adv, num_obstacles=n_obst, max_cycles=max_cycles,
                        device=device, dtype=dtype, seed=seed)


def _actors(env, dtype, hidden=(64, 64, 64), seed=1, shipped=False):
    torch.manual_seed(seed)
    if shipped:
        acts = load_distributed_actors(os.path.join(TRAINED, "ppo_actors_tag_dinno_0_3000.pth"),
                                       lambda: FFReLUNet([12, 64, 64, 64, 5]), 3)
        return [a.to(dtype) for a in acts]
    d0 = env.observation_spaces["adversary_0"].shape[0]
    return [FFReLUNet([d0, *hidden, 5], dtype=dtype) for _ in range(env.n_adv)]


def _on(actors, device):
    import copy
    return [copy.deepcopy(a).to(device) for a in actors]


def _per_cycle(x, n_ep, T, E):
    """[N, R, ...] -> [T, everything else] (max over worlds is taken per cycle)."""
    N = x.shape[0]
    return x.reshape(N, n_ep, T, E, -1).permute(2, 0, 1, 3, 4).reshape(T, -1)


def _cycles(out, n_ep, T, E):
    q = {k: _per_cycle(out[k].double().cpu(), n_ep, T, E) for k in ("obs", "acts", "log_probs", "rtgs")}
    q["pos"] = out["pos"].double().cpu().permute(1, 0, 2, 3, 4).reshape(T, -1)
    return q


def _err(a, b):
    return {k: (a[k] - b[k]).abs().amax(dim=1) for k in a}            # [T] per quantity


def _envelope(e):
    return torch.cummax(e, dim=0).values


def _run_kernel(env, actors, pos0, T, key=7, index=0, noise=1.0):
    n_ep = pos0.shape[0]
    out = tag_rollout.rollout(env, actors, T=T, n_ep=n_ep, gamma=GAMMA, cov_var=COV, noise_scale=noise, key=key,
                              index=index, pos0=pos0, debug=True)
    torch.cuda.synchronize()
    return out


def _oracle(actors, pos0, eps, T, cfg, dtype=torch.float64):
    env = _env(**dict(cfg, dtype=dtype, device="cpu"))
    acts = [a.to("cpu", dtype) for a in _on(actors, "cpu")]
    return replay_tag_rollout(env, acts, pos0.to("cpu", dtype), eps.to("cpu", dtype), T, GAMMA, COV)


def _check_fp64(cfg, actors, n_ep, T):
    env = _env(**cfg)
    pos0 = tag_rollout.reset_positions(env, n_ep)
    out = _run_kernel(env, actors, pos0, T)
    E = env.E
    ref = _oracle(actors, pos0, out["eps"], T, cfg)
    yard = _oracle(actors, torch.nextafter(pos0.cpu(), torch.tensor(float("inf"), dtype=torch.float64)), out["eps"], T, cfg)
    k, o, y = _cycles(out, n_ep, T, E), _cycles(ref, n_ep, T, E), _cycles(yard, n_ep, T, E)
    ek, ey = _err(k, o), _err(y, o)
    worst = 0.0
    for q in k:
        scale = o[q].abs().max().item()
        bound = torch.clamp(10 * _envelope(ey[q]), min=1e-12 * scale)
        assert (ek[q] <= bound).all(), (q, ek[q].tolist(), bound.tolist())
        if q != "rtgs":                                   # an early reward-to-go sums the whole episode
            assert (ek[q][:2] <= 1e-12 * max(scale, 1.0)).all(), (q, ek[q][:2].tolist())
        worst = max(worst, (ek[q] / bound).max().item())
    rk, ro, ry = out["ep_returns"].cpu(), ref["ep_returns"], yard["ep_returns"]
    assert (rk - ro).abs().max() <= max(10 * (ry - ro).abs().max().item(), 1e-12 * ro.abs().max().item())
    print(f"fp64 kernel error / bound, worst over quantities and cycles: {worst:.3g}")
    return out


def test_fp64_kernel_matches_replay_oracle_distinct_actors():
    cfg = dict(E=16, n_obst=8, max_cycles=200)
    _check_fp64(cfg, _on(_actors(_env(**cfg), torch.float64), DEV), n_ep=2, T=50)


def test_fp64_kernel_matches_replay_oracle_shipped_actors():
    """The trained DiNNO predators keep catching the prey, so contacts are exercised."""
    cfg = dict(E=16, n_obst=8, max_cycles=200)
    out = _check_fp64(cfg, _on(_actors(None, torch.float64, shipped=True), DEV), n_ep=2, T=50)
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


def _fp32_ratio(cfg, actors32, T, n_ep, noise=1.0, perturbed_yardstick=False):
    """``perturbed_yardstick``: the torch fp32 error is the larger of the runs from pos0 and from pos0 moved by one fp32
    ulp.  The deterministic trained policy keeps the predators in stiff contact, so when the trajectories first
    amplify a rounding difference depends on where that difference lands; one torch run is then too narrow a sample."""
    env = _env(**dict(cfg, dtype=torch.float32))
    pos0 = tag_rollout.reset_positions(env, n_ep)
    out = _run_kernel(env, actors32, pos0, T, noise=noise)
    E = env.E
    eps = out["eps"] * noise
    ref = _oracle(actors32, pos0, eps, T, cfg)                                         # fp64 oracle, fp32 inputs
    t32 = _oracle(actors32, pos0, eps, T, cfg, dtype=torch.float32)                    # the torch fp32 path
    k, o, t = _cycles(out, n_ep, T, E), _cycles(ref, n_ep, T, E), _cycles(t32, n_ep, T, E)
    ek, et = _err(k, o), _err(t, o)
    if perturbed_yardstick:
        up = torch.nextafter(pos0.cpu(), torch.tensor(float("inf")))
        t2 = _cycles(_oracle(actors32, up, eps, T, cfg, dtype=torch.float32), n_ep, T, E)
        et = {q: torch.maximum(et[q], v) for q, v in _err(t2, o).items()}
    worst = 0.0
    for q in k:
        scale = o[q].abs().max().item()
        floor = 4 * 2.0 ** -23 * scale
        bound = torch.clamp(4 * _envelope(et[q]), min=floor)
        assert (ek[q] <= bound).all(), (q, ek[q].tolist(), bound.tolist())
        worst = max(worst, (ek[q] / torch.clamp(_envelope(et[q]), min=floor)).max().item())
    print(f"fp32 kernel error / torch fp32 error, worst over quantities and cycles: {worst:.3g}")
    return out, worst


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
