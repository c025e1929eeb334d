"""Conv-layer gradients of the float64 cluster kernel (csrc/mnist_cl64.cu) against float64 autograd: every batch split,
u8 and fp32 input rows, full and partial batches, and a fixture built for the max-pool routing: flat image regions,
where the four conv outputs of a pooling window tie and the first maximum wins, and a ReLU-dead channel."""
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


def _flatten_regions(s: Shard, g: int) -> Shard:
    """Coarse grey levels (large equal-valued areas) and, in every other image, a blank band of rows 8 .. 15."""
    x = (s.x // 64) * 64
    x[g % 2::2, :, 8:16, :] = 0
    return Shard(x, s.y, s.norm)


def _problem(B, float_inputs, edge):
    """L nodes, one class each; a node's shard holds B + B // 2 + 1 rows, so the second draw is a partial batch."""
    M = B + B // 2 + 1
    shards = [synthetic_mnist(M, seed=200 + g, classes=[(3 * g) % 10]) for g in range(L)]
    if edge:
        shards = [_flatten_regions(s, g) for g, s in enumerate(shards)]
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
    if edge:
        bc = _slot(pr, "seq.0.bias")
        pr.arena.theta[:, bc.start + 1] = -50.0     # channel 1 is ReLU-dead on every image: its da1 is all zero
    return pr


def _slot(pr, name):
    s = next(s for s in pr.arena.layout.slots if s.name == name)
    return slice(s.offset, s.offset + s.numel)


@pytest.mark.parametrize("edge", [False, True])
@pytest.mark.parametrize("float_inputs", [False, True])
@pytest.mark.parametrize("B", [64, 37])
@pytest.mark.parametrize("nsplit", [1, 2, 4])
def test_conv_grads_match_fp64_oracle(nsplit, B, float_inputs, edge, monkeypatch):
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    pr = _problem(B, float_inputs, edge)
    fz, spec = pr.fused, pr.base_model.spec
    assert fz.cl64 and fz.S == nsplit and fz.x_is_u8 != float_inputs
    norm = () if float_inputs else pr.shards.norm
    wc, bc = _slot(pr, "seq.0.weight"), _slot(pr, "seq.0.bias")
    for step in range(2):                       # full batch, then a partial one
        calls = pr.calls.copy()
        fz.compute_grads()
        for l in range(L):
            rows = ko.batch_rows(pr.shards.sizes, B, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            _, gr = ko.convnet_fp64(pr.arena.theta[l], spec, pr.shards.x[rows], pr.shards.y[rows], *norm)
            g = pr.arena.grad[l]
            torch.testing.assert_close(g[wc], gr[wc], rtol=0, atol=1e-11)
            torch.testing.assert_close(g[bc], gr[bc], rtol=0, atol=1e-11)
            if edge:
                assert torch.all(g[wc].view(3, 25)[1] == 0) and g[bc][1] == 0


@pytest.mark.parametrize("float_inputs", [False, True])
@pytest.mark.parametrize("nsplit", [1, 2, 4])
def test_conv_grads_of_two_launches_are_bitwise_equal(nsplit, float_inputs, monkeypatch):
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    runs = []
    for _ in range(2):
        pr = _problem(37, float_inputs, edge=True)
        assert pr.fused.cl64 and pr.fused.S == nsplit
        out = []
        for _step in range(2):
            pr.fused.compute_grads()
            out.append(torch.cat([pr.arena.grad[:, _slot(pr, "seq.0.weight")], pr.arena.grad[:, _slot(pr, "seq.0.bias")]], 1))
        runs.append(out)
    for a, b in zip(*runs):
        assert torch.equal(a, b)
