"""The fused solo / centralized baselines without a GPU: configuration, refusals, budgets, and the float64 oracle that
the GPU tests compare the kernels with (``tests/test_gpu_local_training.py``)."""
import copy

import pytest
import torch
import yaml

import local_train_oracle as lto
from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.sampler import BatchSchedule
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.experiments import centralized, density_common, dist_mnist_ex
from nn_distributed_training_b200.models import FourierNet, MNISTConvNet
from nn_distributed_training_b200.ops import local_train
from nn_distributed_training_b200.utils.config import ConfigError, validate_experiment

PAPER = "experiments/dist_online_dense_PAPER.yaml"
SOLO = {"train_solo": True, "optimizer": "adam", "lr": 1e-3, "epochs": 2, "train_batch_size": 16,
        "val_batch_size": 10, "verbose": False, "backend": "fused"}


def _paper():
    with open(PAPER) as f:
        return yaml.safe_load(f)


def test_backend_defaults_to_torch():
    conf = validate_experiment(_paper(), "online_density")
    assert conf["experiment"]["individual_training"]["backend"] == "torch"


def test_unknown_backend_is_a_config_error():
    raw = _paper()
    raw["experiment"]["individual_training"]["backend"] = "cuda"
    with pytest.raises(ConfigError, match="individual_training.backend"):
        validate_experiment(raw, "online_density")
    raw["experiment"]["individual_training"]["backend"] = "fused"
    assert validate_experiment(raw, "online_density")["experiment"]["individual_training"]["backend"] == "fused"


def test_fused_on_cpu_raises_in_the_runners():
    shards = [synthetic_mnist(40, seed=g) for g in range(2)]
    with pytest.raises(ValueError, match="CUDA device"):
        local_train.solo_mnist(MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, synthetic_mnist(20, seed=9),
                               torch.device("cpu"), SOLO)
    x = (torch.rand(50, 2) - 0.5) * 1200
    with pytest.raises(ValueError, match="CUDA device"):
        density_common.solo_results(FourierNet([2, 256, 64, 64, 64, 1], scale=0.05), torch.nn.BCELoss(),
                                    [Shard(x, (x[:, 0] > 0).float())], None, torch.device("cpu"), SOLO)


def test_fused_on_cpu_raises_in_train_centralized():
    data = synthetic_mnist(40, seed=0)
    with pytest.raises(ValueError, match="CUDA device"):
        centralized.train_centralized(MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), data, data, torch.device("cpu"),
                                      epochs=1, backend="fused")
    with pytest.raises(ValueError, match="backend"):
        centralized.train_centralized(MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), data, data, torch.device("cpu"),
                                      epochs=1, backend="cudnn")


def test_centralized_cli_takes_a_backend(monkeypatch):
    seen = {}
    monkeypatch.setattr(centralized, "centralized_mnist", lambda path, backend: seen.update(path=path, backend=backend))
    centralized.main(["mnist", "x.yaml", "--backend", "fused"])
    assert seen == {"path": "x.yaml", "backend": "fused"}
    with pytest.raises(SystemExit):
        centralized.main(["mnist", "x.yaml", "--backend", "cudnn"])


def test_budgets_are_epochs_of_batches_per_node():
    # the hetero MNIST split: unequal shards, each with a partial last batch; and a shard smaller than one batch
    sizes = [5923, 6742, 5958, 6131, 5842, 5421, 5918, 6265, 5851, 5949, 37]
    for bs in (64, 100):
        for epochs in (1, 3):
            got = local_train.epoch_budgets(sizes, bs, epochs)
            assert got == [epochs * -(-m // bs) for m in sizes]
            assert got == [epochs * BatchSchedule(m, bs).batches_per_epoch for m in sizes]
    assert local_train.epoch_budgets([37], 64, 2) == [2]


@pytest.mark.parametrize("optimizer", ["sgd", "adam", "adamw"])
def test_host_twin_oracle_equals_the_torch_solo_loop_on_the_same_indices(optimizer, monkeypatch):
    """The autograd oracle of the GPU tests is the torch solo loop itself once both draw the same batches."""
    conf = dict(SOLO, optimizer=optimizer, backend="torch")
    shard, val = synthetic_mnist(45, seed=3), synthetic_mnist(12, seed=4)
    torch.manual_seed(0)
    base = MNISTConvNet(3, 5, 64, dtype=torch.float64)
    ref = lto.HostTwinTrainer(copy.deepcopy(base), torch.nn.NLLLoss(), shard, 16, optimizer, 1e-3, seed=5, node=2)
    ref.run(2 * BatchSchedule(45, 16).batches_per_epoch)
    model = copy.deepcopy(base)
    monkeypatch.setattr(torch, "randperm", lto.feistel_randperm(5, 2))
    dist_mnist_ex.train_solo(model, torch.nn.NLLLoss(), shard, val, torch.device("cpu"), conf)
    assert torch.equal(lto.flat(model), lto.flat(ref.model))


def test_host_twin_oracle_equals_the_torch_density_solo_loop(monkeypatch):
    g = torch.Generator().manual_seed(0)
    x = ((torch.rand(70, 2, generator=g, dtype=torch.float64) - 0.5) * 1200)
    shard = Shard(x, (torch.rand(70, generator=g) < 0.3).double())

    class _Val:          # what train_solo reads of a RandomPoseLidarDataset
        def __init__(self, s):
            self.shard = s
            self.lidar = type("L", (), {"xs": torch.linspace(0, 1, 16).numpy(), "ys": torch.linspace(0, 1, 16).numpy()})

    torch.manual_seed(0)
    base = FourierNet([2, 64, 64, 64, 64, 1], scale=0.05, dtype=torch.float64)
    ref = lto.HostTwinTrainer(copy.deepcopy(base), torch.nn.BCELoss(), shard, 16, "adam", 1e-3, seed=7, node=1,
                              squeeze=True)
    ref.run(2 * BatchSchedule(70, 16).batches_per_epoch)
    model = copy.deepcopy(base)
    monkeypatch.setattr(torch, "randperm", lto.feistel_randperm(7, 1))
    density_common.train_solo(model, torch.nn.BCELoss(), _Val(shard), _Val(shard), torch.device("cpu"),
                              dict(SOLO, backend="torch"))
    assert torch.equal(lto.flat(model), lto.flat(ref.model))
