"""CPU checks of the fused rollout's replay oracle, of ``tag_rollout.supports`` and of the backend option's errors."""
import networkx as nx
import pytest
import torch

from nn_distributed_training_b200.ops import tag_rollout
from nn_distributed_training_b200.rl import PPO, DistPPOProblem, FFReLUNet, SimpleTagEnv
from nn_distributed_training_b200.rl.eval_policy import rollout as eval_rollout
from tag_rollout_oracle import draws_of_split_rollout, replay_tag_rollout


def _problem(E=4, steps=12, tpb=100, seed=0, **kw):
    env = SimpleTagEnv(num_envs=E, num_good=1, num_adversaries=3, num_obstacles=8, max_cycles=steps, seed=seed)
    torch.manual_seed(0)
    return DistPPOProblem(FFReLUNet([12, 16, 16, 5]), FFReLUNet([12, 16, 16, 1]), nx.wheel_graph(3), env,
                          timesteps_per_batch=tpb, max_timesteps_per_episode=steps * 4, gamma=0.99,
                          n_updates_per_iteration=2, lr=3e-4, clip=0.2, **kw)


@pytest.mark.parametrize("steps,max_cycles,tpb", [(12, 12, 100), (12, 7, 200)])
def test_replay_is_bitwise_the_torch_rollout(steps, max_cycles, tpb):
    pr = _problem(steps=steps, tpb=tpb)
    pr.env.max_cycles = max_cycles
    # each predator its own actor
    for i in range(1, 3):
        with torch.no_grad():
            for p in pr.models[i].actor.parameters():
                p.add_(0.1 * i)
    env_state, rng_state = pr.env.gen.get_state(), torch.get_rng_state()
    pr.split_rollout_marl()
    T = min(steps, max_cycles)
    n_ep = -(-tpb // (3 * pr.env.E * T))
    assert pr.curr_obs[0].shape[0] == n_ep * T * pr.env.E
    pr.env.gen.set_state(env_state)
    torch.set_rng_state(rng_state)
    pos0, eps = draws_of_split_rollout(pr.env, 3, n_ep, T)
    out = replay_tag_rollout(pr.env, [pr.models[i].actor for i in range(3)], pos0, eps, T, pr.gamma, pr.cov_var)
    for i in range(3):
        assert torch.equal(out["obs"][i], pr.curr_obs[i])
        assert torch.equal(out["acts"][i], pr.curr_acts[i])
        assert torch.equal(out["log_probs"][i], pr.curr_log_probs[i])
        assert torch.equal(out["rtgs"][i], pr.curr_rtgs[i])
    assert out["ep_returns"].tolist() == pr.logger["batch_rews"]
    assert out["pos"].shape == (n_ep, T, pr.env.E, 4, 2)
    assert torch.equal(out["pos"][-1, -1], pr.env.pos)


def test_supports_accepts_and_rejects():
    env = SimpleTagEnv(num_envs=2, num_obstacles=8)
    assert tag_rollout.supports(env, FFReLUNet([12, 64, 64, 64, 5]))
    assert tag_rollout.supports(env, [FFReLUNet([12, 16, 16, 5]) for _ in range(3)])
    assert tag_rollout.supports(env, FFReLUNet([12, 5]))
    assert not tag_rollout.supports(env, FFReLUNet([12, 65, 5]))                      # too wide
    assert not tag_rollout.supports(env, FFReLUNet([12, 8, 8, 8, 8, 8, 5]))           # 5 hidden layers
    assert not tag_rollout.supports(env, FFReLUNet([12, 16, 4]))                      # not a 5-wide action
    assert not tag_rollout.supports(env, [FFReLUNet([12, 16, 5]), FFReLUNet([12, 32, 5]), FFReLUNet([12, 16, 5])])
    assert not tag_rollout.supports(env, [FFReLUNet([12, 16, 5])] * 2)                # 2 actors for 3 predators
    assert not tag_rollout.supports(env, FFReLUNet([12, 16, 5], dtype=torch.float64))  # dtype differs from the env
    from nn_distributed_training_b200.models.relu_nn import FFTanhNet
    assert not tag_rollout.supports(env, FFTanhNet([12, 16, 5]))
    big = SimpleTagEnv(num_envs=2, num_good=2, num_adversaries=7, num_obstacles=0)    # 9 agents
    assert not tag_rollout.supports(big, FFReLUNet([big.observation_spaces["adversary_0"].shape[0], 16, 5]))
    e7 = SimpleTagEnv(num_envs=2, num_good=1, num_adversaries=7, num_obstacles=2)
    assert tag_rollout.supports(e7, FFReLUNet([e7.observation_spaces["adversary_0"].shape[0], 16, 5]))
    e64 = SimpleTagEnv(num_envs=2, num_good=2, num_adversaries=4, num_obstacles=2, dtype=torch.float64)
    assert tag_rollout.supports(e64, FFReLUNet([18, 64, 5], dtype=torch.float64))


def test_cuda_backend_on_a_cpu_env_raises():
    with pytest.raises(ValueError, match="CUDA device"):
        _problem(rollout_backend="cuda")
    with pytest.raises(ValueError, match="rollout_backend"):
        _problem(rollout_backend="fused")
    env = SimpleTagEnv(num_envs=2, num_obstacles=8, max_cycles=5)
    with pytest.raises(ValueError, match="CUDA device"):
        PPO(FFReLUNet, env, rollout_backend="cuda")
    with pytest.raises(ValueError, match="CUDA device"):
        eval_rollout(FFReLUNet([12, 16, 5]), env, backend="cuda")


def test_cli_flag_reaches_the_problem():
    from nn_distributed_training_b200.rl.train_common import make_problem, parse_args
    args = parse_args(["--num_envs", "2"])
    assert args.rollout == "torch" and make_problem(args)[0].rollout_backend == "torch"
    with pytest.raises(ValueError, match="CUDA device"):
        make_problem(parse_args(["--num_envs", "2", "--rollout", "cuda"]))
    from nn_distributed_training_b200.rl.arguments import get_args
    assert get_args(["--rollout", "cuda"]).rollout == "cuda"
