"""The float64 cluster kernel (csrc/mnist_cl64.cu) with its phases overlapped: W1 copied under the conv, one warp per
owned sample in the head, and dW1 computed alongside the conv-gradient pass.  The whole gradient row and the loss are
checked against float64 autograd for every batch split, u8 and fp32 rows, full and partial batches, and a batch in
which whole clusters hold no valid sample (their head warps see only masked samples)."""
import networkx as nx
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
L = 3


def _problem(B, float_inputs):
    """L nodes, one class each; a node's shard holds B + B // 2 + 1 rows, so the second draw is a partial batch."""
    M = B + B // 2 + 1
    shards = [synthetic_mnist(M, seed=300 + g, classes=[(7 * g + 2) % 10]) for g in range(L)]
    val = synthetic_mnist(64, seed=1)
    if float_inputs:
        shards = [Shard(s.inputs(torch.arange(len(s)), torch.float32), s.y) for s in shards]
        val = Shard(val.inputs(torch.arange(len(val)), torch.float32), val.y)
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": ["validation_loss"],
            "metrics_config": {"evaluate_frequency": 1000},
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}}
    torch.manual_seed(0)
    pr = DistMNISTProblem(nx.cycle_graph(L), MNISTConvNet(3, 5, 64, dtype=torch.float64), torch.nn.NLLLoss(), shards,
                          val, DEV, conf, backend="fused", seed=11)
    for l in range(L):
        pr.arena.theta[l] *= 1.0 + 0.05 * l
    return pr


# B = 20: at nsplit 2 the second cluster, at nsplit 4 the third and fourth hold no valid sample
@pytest.mark.parametrize("float_inputs", [False, True])
@pytest.mark.parametrize("B", [64, 37, 20])
@pytest.mark.parametrize("nsplit", [1, 2, 4])
def test_gradient_row_and_loss_match_fp64_oracle(nsplit, B, float_inputs, monkeypatch):
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    pr = _problem(B, float_inputs)
    fz, spec = pr.fused, pr.base_model.spec
    assert fz.cl64 and fz.S == nsplit and fz.x_is_u8 != float_inputs
    norm = () if float_inputs else pr.shards.norm
    for step in range(2):                       # full batch, then a partial one
        calls = pr.calls.copy()
        loss = fz.compute_grads().clone()
        for l in range(L):
            rows = ko.batch_rows(pr.shards.sizes, B, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            lr, gr = ko.convnet_fp64(pr.arena.theta[l], spec, pr.shards.x[rows], pr.shards.y[rows], *norm)
            torch.testing.assert_close(loss[l].double(), lr, rtol=1e-6, atol=1e-7)   # loss partials are stored as float
            torch.testing.assert_close(pr.arena.grad[l], gr, rtol=0, atol=1e-11)


@pytest.mark.parametrize("float_inputs", [False, True])
@pytest.mark.parametrize("nsplit", [1, 2, 4])
def test_two_launches_are_bitwise_equal(nsplit, float_inputs, monkeypatch):
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    runs = []
    for _ in range(2):
        pr = _problem(20, float_inputs)
        assert pr.fused.cl64 and pr.fused.S == nsplit
        out = []
        for _step in range(2):
            loss = pr.fused.compute_grads().clone()
            out.append((loss, pr.arena.grad.clone()))
        runs.append(out)
    for (la, ga), (lb, gb) in zip(*runs):
        assert torch.equal(la, lb) and torch.equal(ga, gb)
