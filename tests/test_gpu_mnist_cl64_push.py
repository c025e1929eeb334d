"""The float64 cluster kernel (csrc/mnist_cl64.cu) against recorded outputs: its gradient partial rows and loss partials
must stay bitwise what `tests/golden/cl64_grads.npz` holds, at every batch split, at full and partial batches (at B = 37
some owner CTAs hold only invalid samples), for u8 and fp32 input rows and at 3 and 10 nodes.

A partial row is 28,440 doubles, so the fixture keeps the SHA-256 of each parameter slot of each row (a bitwise record
that names the slot that moved) and the float32 loss partials themselves.  `scripts/record_cl64_golden.py` wrote it."""
import hashlib
import itertools
import os

import networkx as nx
import numpy as np
import pytest
import torch

from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cl64_grads.npz")
STEPS = 2
CONFIGS = list(itertools.product([1, 2, 4], [64, 37], ["u8", "f32"], [3, 10]))   # nsplit, B, input rows, nodes


def key(nsplit, B, rows, L):
    return f"s{nsplit}_b{B}_{rows}_l{L}"


def run(nsplit, B, rows, L):
    """STEPS launches of the kernel on a fixed problem: (loss partials [STEPS, L, S] float32, slot digests [STEPS, L, S,
    slots, 32] uint8).  NNDT_TC_SPLIT must be set to nsplit.  A node's shard holds B + B // 2 + 1 rows, so the second
    draw is a partial batch."""
    M = B + B // 2 + 1
    shards = [synthetic_mnist(M, seed=100 + g, classes=[g % 10]) for g in range(L)]
    val = synthetic_mnist(64, seed=1)
    if rows == "f32":
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
    fz = pr.fused
    assert fz.cl64 and fz.S == nsplit and fz.x_is_u8 == (rows == "u8")
    slots = pr.arena.layout.slots
    losses, digests = [], []
    for _ in range(STEPS):
        fz.compute_grads()
        losses.append(fz.loss_part.cpu().numpy().copy())
        g = fz.grad_part.cpu().numpy()
        digests.append([[[np.frombuffer(hashlib.sha256(np.ascontiguousarray(g[l, s, t.offset: t.offset + t.numel]).tobytes())
                                        .digest(), np.uint8) for t in slots] for s in range(nsplit)] for l in range(L)])
    return np.stack(losses), np.array(digests, dtype=np.uint8), [t.name for t in slots]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit,B,rows,L", CONFIGS)
def test_matches_recorded_outputs(nsplit, B, rows, L, golden, monkeypatch):
    """Two launches from the same inputs, each bitwise equal to the recorded kernel outputs."""
    monkeypatch.setenv("NNDT_TC_SPLIT", str(nsplit))
    k = key(nsplit, B, rows, L)
    want_loss, want_dig = golden[k + "_loss"], golden[k + "_digest"]
    for _ in range(2):
        loss, dig, names = run(nsplit, B, rows, L)
        assert np.array_equal(loss.view(np.uint32), want_loss.view(np.uint32)), (loss, want_loss)
        bad = {(st, l, s, names[t]) for st, l, s, t in zip(*np.nonzero((dig != want_dig).any(-1)))}
        assert not bad, f"gradient slots differ from the recorded ones (step, node, split, slot): {sorted(bad)}"
