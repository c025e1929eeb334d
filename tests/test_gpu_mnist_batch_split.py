"""The fp32 batch-split training kernel ``mnist_kernel<SPB, 768, true>`` (csrc/mnist.cu, mnist_device.cuh) against the
float64 oracle at every samples-per-CTA instantiation.

The paper net in fp32 runs this kernel whenever the batch is above 64 (or ``mnist_kernel`` is not ``tc``): the solo
and individual-training runs at batch 100 among them.  ``choose_spb`` picks 4..8 samples per CTA from the node count;
the instantiations with 5, 6 and 7 are the ones that zero-pad the MMA operands to 8 samples.  The yardstick is the
one of ``test_cluster_kernels_match_fp64_oracle_at_every_instantiation``: the 3xTF32 kernel's error is at most 0.1x
that of a 1xTF32 emulation of the three fc1-sized contractions, per tensor and per 16 x 8 block.

Both oracles take the max-pool argmax from the conv as an fp32 kernel evaluates it (``pool_f32``).  At batch 100 the
first batch of node 0 holds a pool window whose two largest conv outputs differ by 7e-8, less than fp32 resolves: the
kernel, like fp32 autograd, routes that cell's gradient to the other position, and that alone puts the conv-weight
gradient at 0.17x the yardstick's error when measured against the fp64 routing (tests/test_kernel_oracles.py)."""
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
METRICS = ["forward_pass_count", "validation_loss", "top1_accuracy"]


def _problem(L, B, spb, float_rows):
    """bench.py's data layout: one class per node, a different network per node (``theta[l] *= 1 + 0.03 l``), and
    ``B + B // 2 + 1`` rows per node, so draw 0 is a full batch, draw 1 a partial one and draw 2 opens epoch 1."""
    M = B + B // 2 + 1
    shards = [synthetic_mnist(M, seed=100 + g, classes=[g % 10]) for g in range(L)]
    if float_rows:
        shards = [Shard(s.inputs(torch.arange(len(s)), torch.float32), s.y) for s in shards]
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": METRICS,
            "metrics_config": {"evaluate_frequency": 1000}, "samples_per_cta": spb, "mnist_kernel": "mma",
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2,
                                 "profile": False}}
    torch.manual_seed(0)
    pr = DistMNISTProblem(nx.cycle_graph(L), MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards,
                          synthetic_mnist(16, seed=1), DEV, conf, backend="fused", seed=7)
    for l in range(L):
        pr.arena.theta[l] *= 1.0 + 0.03 * l
    return pr


def _run_and_compare(L, B, spb, float_rows, steps=3):
    pr = _problem(L, B, spb, float_rows)
    fz, spec = pr.fused, pr.base_model.spec
    assert not fz.tc and not fz.generic and fz.spb == spb and fz.S == -(-B // spb)
    mean, std = pr.shards.norm if pr.shards.norm is not None else (0.0, 1.0)
    pad = ko.padding_mask(spec, fz.n_pad, DEV)
    worst = {}
    for step in range(steps):               # full batch, partial batch, first batch of the next epoch
        calls = pr.calls.copy()
        ko.poison_partials(fz, spec)
        loss = fz.compute_grads().clone()
        assert not fz.grad_part[:, :, pad].any(), "the kernel wrote the arena padding"
        assert torch.isfinite(fz.loss_part).all(), "a slice left its loss partial unwritten"
        assert torch.isfinite(pr.arena.grad).all(), "a slice left part of its gradient row unwritten"
        for l in range(L):
            rows = ko.batch_rows(pr.shards.sizes, B, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            x, y, th = pr.shards.x[rows], pr.shards.y[rows], pr.arena.theta[l]
            lr, gr = ko.convnet_fp64(th, spec, x, y, mean, std, pool_f32=True)
            gt = ko.convnet_fp64(th, spec, x, y, mean, std, tf32_fc1=True, pool_f32=True)[1]
            assert abs(loss[l].item() - lr.item()) <= 1e-5 * abs(lr.item()), (l, step, loss[l].item(), lr.item())
            rat = ko.assert_close_to_oracle(pr.arena.grad[l].double(), gr, gt, ko.CONVNET_FRAC, spec=spec)
            for k, v in rat.items():
                worst[k] = max(worst.get(k, 0.0), *v)
    rows_kind = "f32" if float_rows else "u8"
    print(f"\nRATIO mnist_kernel<{spb}> B={B} {rows_kind}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("float_rows", [False, True], ids=["u8", "f32"])
@pytest.mark.parametrize("B", [100, 37, 8])
@pytest.mark.parametrize("spb", [4, 5, 6, 7, 8])
def test_batch_split_kernel_matches_fp64_oracle_at_every_spb(spb, B, float_rows):
    _run_and_compare(3, B, spb, float_rows)


def test_batch_split_kernel_matches_fp64_oracle_over_several_waves():
    """Batch 1000 at 8 samples per CTA: 125 slices per node, 375 CTAs, several waves of the SMs."""
    _run_and_compare(3, 1000, 8, False)
