"""The float64 cluster kernel (csrc/mnist_cl64.cu) beyond what test_gpu_mnist.py checks: bitwise determinism, fp32
input rows at every instantiation, and that the benchmark's clusters fit in one wave on an H100 SXM."""
import networkx as nx
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.ops import load_ext
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _problem(L, B, float_inputs=False):
    """L nodes, one class each; a node's shard holds B + B // 2 + 1 rows, so the second draw is a partial batch."""
    M = B + B // 2 + 1
    shards = [synthetic_mnist(M, seed=100 + g, classes=[g % 10]) for g in range(L)]
    val = synthetic_mnist(64, seed=1)
    if float_inputs:
        shards = [Shard(s.inputs(torch.arange(len(s)), torch.float32), s.y) for s in shards]
        val = Shard(val.inputs(torch.arange(len(val)), torch.float32), val.y)
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": ["validation_loss"],
            "metrics_config": {"evaluate_frequency": 1000},
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}}
    torch.manual_seed(0)
    pr = DistMNISTProblem(nx.cycle_graph(L), MNISTConvNet(3, 5, 64, dtype=torch.float64), torch.nn.NLLLoss(), shards,
                          val, DEV, conf, backend="fused", seed=7)
    for l in range(L):
        pr.arena.theta[l] *= 1.0 + 0.03 * l
    return pr


@pytest.mark.parametrize("nsplit", [1, 2, 4])
def test_two_launches_are_bitwise_equal(nsplit, monkeypatch):
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    runs = []
    for _ in range(2):
        pr = _problem(3, 64)
        assert pr.fused.cl64 and pr.fused.S == nsplit
        out = []
        for step in range(2):
            loss = pr.fused.compute_grads().clone()
            out.append((loss, pr.arena.grad.clone()))
        runs.append(out)
    for (la, ga), (lb, gb) in zip(*runs):
        assert torch.equal(la, lb) and torch.equal(ga, gb)


@pytest.mark.parametrize("nsplit", [1, 2, 4])
@pytest.mark.parametrize("B", [64, 37])
def test_float_inputs_match_fp64_oracle(B, nsplit, monkeypatch):
    """fp32 rows: normalised doubles in shared memory at 16 and 32 samples per cluster, read from L2 at 64."""
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    L = 3
    pr = _problem(L, B, float_inputs=True)
    fz, spec = pr.fused, pr.base_model.spec
    assert fz.cl64 and fz.S == nsplit and not fz.x_is_u8
    for step in range(2):
        calls = pr.calls.copy()
        loss = fz.compute_grads().clone()
        for l in range(L):
            rows = ko.batch_rows(pr.shards.sizes, B, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            lr, gr = ko.convnet_fp64(pr.arena.theta[l], spec, pr.shards.x[rows], pr.shards.y[rows])
            torch.testing.assert_close(loss[l], lr, rtol=1e-6, atol=1e-7)       # loss partials are stored as float
            torch.testing.assert_close(pr.arena.grad[l], gr, rtol=1e-9, atol=1e-11)


def test_benchmark_clusters_fit_in_one_wave():
    """bench.py runs 10 nodes x 2 batch splits: all 20 clusters must be resident at once on a 132-SM H100."""
    if torch.cuda.get_device_properties(DEV).multi_processor_count != 132:
        pytest.skip("cluster placement depends on the GPC layout of an H100 SXM")
    pr = _problem(10, 64)
    assert pr.fused.cl64 and pr.fused.S == 2
    assert load_ext(required=True).mnist_cl64_max_clusters(pr.fused.S) >= 10 * pr.fused.S
