"""What the PPO update kernels (ops/ppo_update.py) accept, and how ``update_backend`` / ``--update`` reach the problem.
No GPU needed: the checks run before any launch."""
import networkx as nx
import pytest
import torch

from nn_distributed_training_b200.models.relu_nn import FFTanhNet
from nn_distributed_training_b200.ops import ppo_update
from nn_distributed_training_b200.rl import PPO, DistPPOProblem, FFReLUNet, SimpleTagEnv


def _pair(obs=12, hidden=(64, 64, 64), dtype=None, act=5):
    return FFReLUNet([obs, *hidden, act], dtype=dtype), FFReLUNet([obs, *hidden, 1], dtype=dtype)


@pytest.mark.parametrize("hidden", [(), (32,), (64, 64, 64), (64, 64, 64, 64), (1, 7, 64)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("obs", [8, 12, 64])
def test_supported_shapes(hidden, dtype, obs):
    a, c = _pair(obs, hidden, dtype)
    assert ppo_update.supports(a, c) and ppo_update.unsupported_reason([a] * 3, [c] * 3) is None


@pytest.mark.parametrize("make,reason", [
    (lambda: _pair(hidden=(64,) * 5), "hidden layers"),                             # 5 hidden layers
    (lambda: _pair(hidden=(65,)), "width"),                                          # too wide
    (lambda: _pair(obs=65), "width"),
    (lambda: _pair(act=4), "output"),                                                # not a 5-wide action
    (lambda: (FFReLUNet([12, 16, 5]), FFReLUNet([12, 16, 2])), "output"),            # 2-wide critic
    (lambda: (FFReLUNet([12, 16, 5]), FFReLUNet([13, 16, 1])), "input widths"),
    (lambda: (FFTanhNet([12, 16, 5]), FFReLUNet([12, 16, 1])), "not a ReLU MLP"),
    (lambda: (FFReLUNet([12, 16, 5]), FFTanhNet([12, 16, 1])), "not a ReLU MLP"),
    (lambda: _pair(dtype=torch.float16), "dtype"),
    (lambda: (FFReLUNet([12, 16, 5]), FFReLUNet([12, 16, 1], dtype=torch.float64)), "dtype"),
    (lambda: (torch.nn.Sequential(torch.nn.Linear(12, 5)), FFReLUNet([12, 1])), "not a ReLU MLP"),
])
def test_unsupported_configurations_name_the_reason(make, reason):
    a, c = make()
    assert not ppo_update.supports(a, c)
    assert reason in ppo_update.unsupported_reason(a, c)


def test_biases_node_counts_and_shapes_across_nodes():
    a, c = _pair(hidden=(16,))
    a.seq[0].bias = None
    assert "biases" in ppo_update.unsupported_reason(a, c)
    a, c = _pair(hidden=(16,))
    assert "nodes" in ppo_update.unsupported_reason([a] * 9, [c] * 9)
    assert "nodes" in ppo_update.unsupported_reason([a] * 3, [c] * 2)
    a2, _ = _pair(hidden=(32,))
    assert "differ in shape" in ppo_update.unsupported_reason([a, a2, a], [c] * 3)


def test_require_needs_cuda_and_names_the_reason():
    a, c = _pair(hidden=(16,))
    with pytest.raises(ValueError, match="CUDA device"):
        ppo_update.require(a, c)
    with pytest.raises(ValueError, match="CUDA device"):
        ppo_update.advantages(c, torch.zeros(1, 4, 12), torch.zeros(1, 4))


def test_shape_errors_name_the_tensors_device():
    """A wrongly placed batch, output or workspace tensor is named with its device as ``cuda:1`` / ``cpu`` reads,
    not as the ``device(type=...)`` a tuple would print."""
    dev = torch.device("cuda", 0)
    for check in (ppo_update._out, ppo_update._batch):
        with pytest.raises(ValueError, match=r"out: expected .* on cuda:0, got \(8, 40\) torch.float64 on cpu$"):
            check("out", torch.zeros(8, 40, dtype=torch.float64), (8, 40), torch.float64, dev)


def _problem(**kw):
    env = SimpleTagEnv(num_envs=2, num_good=1, num_adversaries=3, num_obstacles=8, max_cycles=5)
    return DistPPOProblem(FFReLUNet([12, 16, 5]), FFReLUNet([12, 16, 1]), nx.wheel_graph(3), env,
                          timesteps_per_batch=30, max_timesteps_per_episode=20, **kw)


def test_update_backend_defaults_to_torch_and_validates():
    pr = _problem()
    assert pr.update_backend == "torch" and pr.batched_grads is None
    with pytest.raises(ValueError, match="update_backend"):
        _problem(update_backend="fused")
    with pytest.raises(ValueError, match="CUDA device"):
        _problem(update_backend="cuda")
    env = SimpleTagEnv(num_envs=2, num_obstacles=8, max_cycles=5)
    assert PPO(FFReLUNet, env).update_backend == "torch"
    with pytest.raises(ValueError, match="update_backend"):
        PPO(FFReLUNet, env, update_backend="fused")
    with pytest.raises(ValueError, match="CUDA device"):
        PPO(FFReLUNet, env, update_backend="cuda")


def test_update_flag_reaches_the_problem():
    from nn_distributed_training_b200.rl.arguments import get_args
    from nn_distributed_training_b200.rl.train_common import make_problem, parse_args
    args = parse_args(["--num_envs", "2"])
    assert args.update == "torch" and make_problem(args)[0].update_backend == "torch"
    with pytest.raises(ValueError, match="CUDA device"):
        make_problem(parse_args(["--num_envs", "2", "--update", "cuda"]))
    with pytest.raises(SystemExit):
        parse_args(["--update", "fused"])
    assert get_args(["--update", "cuda"]).update == "cuda" and get_args([]).update == "torch"
