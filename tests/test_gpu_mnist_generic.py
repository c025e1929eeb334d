"""The generic CUDA-core training kernel ``convnet_generic_kernel<T, KS, SPB, true>`` (csrc/mnist_generic.cu) against
the float64 oracle at every instantiation and at the shape edges.

The kernel trains every float64 problem the cl64 cluster kernel does not take (batch above 64, any shape other than
the paper's) and every fp32 shape other than the paper's (3, 5, 64).  ``FusedMnist`` picks 8 samples per CTA when
``L * ceil(B / 8)`` fills half the SMs and the carve fits in 200 KB, 4 otherwise; ``NNDT_GENERIC_SPB`` forces the
choice, so the cases below reach both at a few nodes.  The shapes cover one and eight filters, both kernel sizes,
linear widths 1 .. 128 (odd ones too) and the conv-gradient partition counts ``512 / (F KS^2 + F)`` at their extremes:
2 at (8, 5, .) and 51 at (1, 3, .).

float64 is held to rtol 1e-9 / atol 1e-11 (losses to 1e-6: the loss partials are stored as float).  fp32 is held to
``TF32_POINT_FRAC`` of the yardstick ``convnet_tf32_point`` per tensor and per 16 x 8 block; both fp32 oracles take
the max-pool argmax from the conv as an fp32 kernel evaluates it (``pool_f32``)."""
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
F32, F64 = torch.float32, torch.float64

# id -> (dtype, (F, KS, LW), B, rows, samples per CTA).  The first eight are one per training instantiation.
CASES = {
    "f32_k5_s4": (F32, (2, 5, 33), 37, "u8", 4),
    "f32_k5_s8": (F32, (8, 5, 128), 37, "u8", 8),                  # npart 2
    "f32_k3_s4": (F32, (1, 3, 1), 37, "f32", 4),                   # npart 51, linear width 1
    "f32_k3_s8": (F32, (8, 3, 100), 100, "u8_norm", 8),
    "f64_k5_s4": (F64, (3, 5, 64), 37, "u8", 4),                   # the paper's net past the cl64 kernel
    "f64_k5_s8": (F64, (3, 5, 64), 64, "f32", 8),
    "f64_k3_s4": (F64, (8, 3, 128), 8, "u8", 4),
    "f64_k3_s8": (F64, (1, 3, 10), 9, "f32", 8),
    "f32_1x5x10_B1": (F32, (1, 5, 10), 1, "u8", 4),
    "f32_8x5x1_B1": (F32, (8, 5, 1), 1, "u8", 8),
    "f32_8x3x128_B8": (F32, (8, 3, 128), 8, "f32", 8),
    "f32_1x3x100_B4": (F32, (1, 3, 100), 4, "u8_norm", 4),
    "f32_2x5x128_B3": (F32, (2, 5, 128), 3, "f32", 8),
    "f64_1x5x1_B3": (F64, (1, 5, 1), 3, "u8_norm", 8),
    "f64_2x3x33_B5": (F64, (2, 3, 33), 5, "u8", 4),
    "f64_8x5x100_B100": (F64, (8, 5, 100), 100, "f32", 4),         # npart 2 in float64
    "f64_1x3x1_B37": (F64, (1, 3, 1), 37, "u8", 8),                # npart 51 in float64
    "f64_8x5x10_B100": (F64, (8, 5, 10), 100, "u8_norm", 4),
}


def _rows(shard, kind):
    """``u8``: the shard as it is; ``f32``: its normalised inputs as float rows; ``u8_norm``: uint8 with a
    normalisation of its own."""
    if kind == "f32":
        return Shard(shard.inputs(torch.arange(len(shard)), torch.float32), shard.y)
    if kind == "u8_norm":
        return Shard(shard.x, shard.y, (0.5, 0.25))
    return shard


def _problem(L, dtype, shape, B, rows):
    """bench.py's data layout: one class per node, a different network per node (``theta[l] *= 1 + 0.03 l``), and
    ``B + B // 2 + 1`` rows per node, so draw 0 is a full batch, draw 1 a partial one and draw 2 opens epoch 1.  b1 is
    made positive so that no net has every fc1 unit off, which would zero every gradient before fc2's at width 1."""
    M = B + B // 2 + 1
    shards = [_rows(synthetic_mnist(M, seed=100 + g, classes=[g % 10]), rows) for g in range(L)]
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": METRICS,
            "metrics_config": {"evaluate_frequency": 1000},
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2,
                                 "profile": False}}
    torch.manual_seed(0)
    pr = DistMNISTProblem(nx.cycle_graph(L), MNISTConvNet(*shape, dtype=dtype), torch.nn.NLLLoss(), shards,
                          synthetic_mnist(16, seed=1), DEV, conf, backend="fused", seed=7)
    o, (lw,) = ko.slots(pr.base_model.spec)[3]
    for l in range(L):
        pr.arena.theta[l] *= 1.0 + 0.03 * l
        pr.arena.theta[l, o: o + lw] = pr.arena.theta[l, o: o + lw].abs() + 0.1
    return pr


def _run_and_compare(monkeypatch, L, dtype, shape, B, rows, spb, force_spb=None, steps=3):
    """Build the problem with ``NNDT_GENERIC_SPB=force_spb`` (unset: the selector's choice), assert the kernel and
    samples per CTA it runs, then compare ``steps`` launches with the oracle node by node."""
    monkeypatch.setenv("NNDT_MNIST_CL64", "0")
    if force_spb is None:
        monkeypatch.delenv("NNDT_GENERIC_SPB", raising=False)
    else:
        monkeypatch.setenv("NNDT_GENERIC_SPB", str(force_spb))
    pr = _problem(L, dtype, shape, B, rows)
    fz, spec = pr.fused, pr.base_model.spec
    assert fz.generic and not fz.tc and not fz.cl64 and fz.dtype == dtype
    assert fz.spb == spb and fz.S == -(-B // spb), (fz.spb, fz.S)
    mean, std = pr.shards.norm if pr.shards.norm is not None else (0.0, 1.0)
    pad = ko.padding_mask(spec, fz.n_pad, DEV)
    worst, alive = {}, set()
    for step in range(steps):               # full batch, partial batch, first batch of the next epoch
        calls, dev_calls = pr.calls.copy(), fz.calls.clone()
        ko.poison_partials(fz, spec)
        loss = fz.compute_grads().clone()
        assert not fz.grad_part[:, :, pad].any(), "the kernel wrote the arena padding"
        assert torch.isfinite(fz.grad_part[:, :, ~pad]).all(), "a slice left part of its partial row unwritten"
        assert torch.isfinite(fz.loss_part).all(), "a slice left its loss partial unwritten"
        assert torch.equal(fz.calls, dev_calls + 1), "every node's draw counter advances once per launch"
        assert not fz.arrive.any(), "the last CTA of a node resets its arrival counter"
        for l in range(L):
            rows_l = ko.batch_rows(pr.shards.sizes, B, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            x, y, th = pr.shards.x[rows_l], pr.shards.y[rows_l], pr.arena.theta[l]
            got = pr.arena.grad[l]
            if dtype == F64:
                lr, gr = ko.convnet_fp64(th, spec, x, y, mean, std)
                assert abs(loss[l].item() - lr.item()) <= 1e-6 * abs(lr.item()), (l, step, loss[l].item(), lr.item())
                torch.testing.assert_close(got, gr, rtol=1e-9, atol=1e-11)
                err = ((got - gr).abs() / (1e-11 + 1e-9 * gr.abs())).max().item()
                worst["tol"] = max(worst.get("tol", 0.0), err)
            else:
                lr, gr = ko.convnet_fp64(th, spec, x, y, mean, std, pool_f32=True)
                gt = ko.convnet_tf32_point(th, spec, x, y, mean, std)[1]
                assert abs(loss[l].item() - lr.item()) <= 1e-5 * abs(lr.item()), (l, step, loss[l].item(), lr.item())
                rat = ko.assert_close_to_oracle(got.double(), gr, gt, ko.TF32_POINT_FRAC, spec=spec)
                for k, v in rat.items():
                    worst[k] = max(worst.get(k, 0.0), *v)
            alive |= {i for i, t in enumerate(ko.unflatten(gr, spec)) if t.abs().max() > 0}
    assert alive == set(range(6)), f"tensors {set(range(6)) - alive} of the oracle's gradient are zero throughout"
    what = "float" if dtype == F32 else "double"
    print(f"\nRATIO convnet_generic_kernel<{what}, {shape[1]}, {spb}> {shape} B={B} {rows}: "
          + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("case", list(CASES))
def test_generic_kernel_matches_fp64_oracle(case, monkeypatch):
    dtype, shape, B, rows, spb = CASES[case]
    _run_and_compare(monkeypatch, 3, dtype, shape, B, rows, spb, force_spb=spb)


def test_cases_run_every_training_instantiation():
    """Each case asserts the samples per CTA it runs, so the table covers all eight ``(T, KS, SPB)`` training
    instantiations; the first eight cases are one per instantiation."""
    ran = {(dtype, shape[1], spb) for dtype, shape, _, _, spb in CASES.values()}
    want = {(t, ks, spb) for t in (F32, F64) for ks in (3, 5) for spb in (4, 8)}
    assert ran == want
    assert {(d, s[1], spb) for d, s, _, _, spb in list(CASES.values())[:8]} == want


def test_samples_per_cta_that_do_not_fit_are_refused(monkeypatch):
    """float64 (8, 3, 128) carves more than 200 KB at 8 samples per CTA: a request for 8 runs 4."""
    from nn_distributed_training_b200.ops import load_ext
    assert load_ext(required=True).convnet_generic_smem_bytes(8, 3, 128, 1, 8) > 200 * 1024
    _run_and_compare(monkeypatch, 3, F64, (8, 3, 128), 37, "u8", 4, force_spb=8, steps=1)


@pytest.mark.parametrize("dtype,shape", [(F64, (3, 5, 64)), (F32, (8, 5, 128))], ids=["f64_3x5x64", "f32_8x5x128"])
def test_generic_kernel_over_several_waves(dtype, shape, monkeypatch):
    """Batch 1000 at 8 samples per CTA on 3 nodes: 125 slices per node, 375 CTAs, several waves of the SMs, every
    draw counter still advanced exactly once per launch."""
    _run_and_compare(monkeypatch, 3, dtype, shape, 1000, "u8", 8, force_spb=8)


def test_selector_picks_8_samples_per_cta_at_the_paper_geometry(monkeypatch):
    """The reference's PAPER geometry in float64: 10 nodes at batch 100 make 10 x 13 = 130 CTAs at 8 samples per
    CTA, at least half of the SMs, so the selector itself picks ``convnet_generic_kernel<double, 5, 8, true>``."""
    if torch.cuda.get_device_properties(DEV).multi_processor_count != 132:
        pytest.skip("the node count is chosen for the 132 SMs of an H100 SXM")
    _run_and_compare(monkeypatch, 10, F64, (3, 5, 64), 100, "u8", 8, force_spb=None, steps=2)
