"""The evaluation kernels against the float64 oracle ``kernel_oracles.convnet_fp64_eval``, per node and per sample.

``mnist_kernel<8, 768, false>`` (csrc/mnist.cu) evaluates the paper net in fp32; ``convnet_generic_kernel<T, KS, SPB,
false>`` (csrc/mnist_generic.cu) every fp64 problem (the cl64 problems and the bench headline's ``top1_after_rounds``
included) and every other shape.  Their per-sample losses and correctness flags are ``validation_loss``,
``top1_accuracy`` and ``validation_as_vector``.  A CTA walks the sample chunks ``blockIdx.x, blockIdx.x + gridDim.x,
...``: the validation sizes here give a CTA several chunks with a partial last one, and one run gives every node a
single CTA that walks all of them."""
import math

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
METRICS = ["validation_loss", "top1_accuracy"]
F64, F32 = torch.float64, torch.float32
# kernel -> (MNISTConvNet shape, dtype); "mnist_eval" is the only one that does not run the generic kernel
KERNELS = {"mnist_eval": ((3, 5, 64), F32), "generic_f64_paper": ((3, 5, 64), F64),
           "generic_f32_8x3x128": ((8, 3, 128), F32), "generic_f64_8x3x128": ((8, 3, 128), F64),
           "generic_f32_2x5x32": ((2, 5, 32), F32), "generic_f64_2x5x32": ((2, 5, 32), F64)}


def _rows(shard, kind):
    """``u8``: the shard as it is (uint8, normalised in-kernel); ``f32``: the normalised inputs as float rows;
    ``u8_norm``: uint8 with a normalisation of its own; ``f32_raw``: float rows of ``x / 255``, unnormalised."""
    if kind == "u8":
        return shard
    if kind == "u8_norm":
        return Shard(shard.x, shard.y, (0.5, 0.25))
    if kind == "f32_raw":
        return Shard(shard.x.float() / 255.0, shard.y)
    return Shard(shard.inputs(torch.arange(len(shard)), torch.float32), shard.y)


def _problem(kernel, V, L=3, val_rows="u8", train_rows="u8", val=None, B=8, M=20, val_batch=64):
    shape, dtype = KERNELS[kernel]
    shards = [_rows(synthetic_mnist(M, seed=100 + g), train_rows) for g in range(L)]
    val = _rows(val if val is not None else synthetic_mnist(V, seed=4), val_rows)
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": val_batch, "metrics": METRICS,
            "metrics_config": {"evaluate_frequency": 1000},
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2,
                                 "profile": False}}
    torch.manual_seed(0)
    pr = DistMNISTProblem(nx.cycle_graph(L), MNISTConvNet(*shape, dtype=dtype), torch.nn.NLLLoss(), shards, val,
                          DEV, conf, backend="fused", seed=7)
    assert pr.fused.generic == (kernel != "mnist_eval") and pr.dtype == dtype
    for l in range(L):                      # a different network per node, so a node mix-up cannot go unnoticed
        pr.arena.theta[l] *= 1.0 + 0.03 * l
    return pr


def _validate(pr):
    """``validate()`` after filling its outputs with values no kernel writes: every ``[L, V]`` entry must be
    written."""
    fz = pr.fused
    fz.val_loss.fill_(float("nan"))
    fz.val_correct.fill_(255)
    loss, _ = fz.validate()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all(), "unwritten per-sample losses"
    assert ((fz.val_correct == 0) | (fz.val_correct == 1)).all(), "unwritten correctness flags"
    return loss.clone(), fz.val_correct.clone().bool()


def _oracle(pr, l, tf32_fc1=False):
    mean, std = pr.val.norm if pr.val.norm is not None else (0.0, 1.0)
    return ko.convnet_fp64_eval(pr.arena.theta[l], pr.base_model.spec, pr.val.x, pr.val.y, mean, std,
                                tf32_fc1=tf32_fc1)


def _margin(z):
    top = z.topk(2, dim=1).values
    return top[:, 0] - top[:, 1]


def _check(pr, kernel, tag=""):
    """Every node's per-sample losses and flags against the oracle; prints the worst fp64 error as a fraction of
    the tolerance, or the fp32 ambiguous flags (and the worst ratio to the 1xTF32 yardstick of ``mnist_eval``)."""
    loss, ok = _validate(pr)
    dtype = KERNELS[kernel][1]
    worst, ambiguous = 0.0, 0
    for l in range(pr.placement.L):
        nll, z = _oracle(pr, l)
        got = loss[l].double()
        ref_ok = z.argmax(1) == pr.val.y
        clear = _margin(z) > (1e-9 if dtype == F64 else 1e-4)
        assert torch.equal(ok[l][clear], ref_ok[clear]), (l, (ok[l] != ref_ok).nonzero().flatten().tolist())
        if dtype == F64:
            torch.testing.assert_close(got, nll, rtol=1e-9, atol=1e-11)
            worst = max(worst, ((got - nll).abs() / (1e-11 + 1e-9 * nll.abs())).max().item())
        else:
            ambiguous += int((~clear).sum())
            if kernel == "mnist_eval":
                yard = _oracle(pr, l, tf32_fc1=True)[0]
                rat = ko.assert_close_to_oracle({"loss": got}, {"loss": nll}, {"loss": yard}, ko.CONVNET_FRAC,
                                                block=(128, 1))
                worst = max(worst, *rat["loss"])
            else:
                torch.testing.assert_close(got, nll, rtol=1e-5, atol=1e-7)
    what = (f"worst error {worst:.2e} of the tolerance" if dtype == F64 else f"ambiguous flags {ambiguous}"
            + (f", worst ratio {worst:.2e}" if kernel == "mnist_eval" else ""))
    print(f"\nEVAL {kernel} {tag}: {what}")


@pytest.mark.parametrize("val_rows", ["u8", "f32"])
@pytest.mark.parametrize("V", [1, 7, 8, 203, 1003])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_eval_kernel_matches_fp64_oracle(kernel, V, val_rows):
    """At 3 nodes V = 1003 gives each CTA several 8-sample chunks, the last of them partial."""
    pr = _problem(kernel, V, val_rows=val_rows)
    _check(pr, kernel, f"V={V} {val_rows}")


def test_generic_eval_runs_both_samples_per_cta_branches():
    """The samples per CTA ``launch_generic_eval`` picks for the generic shapes above: fp64 (8, 3, 128) carves too much
    shared memory for 8 samples and takes the 4-sample branch, every other shape the 8-sample one.  So the case above
    runs both instantiations of the evaluation kernel."""
    from nn_distributed_training_b200.ops import load_ext
    ext = load_ext(required=True)
    got = {k: ext.convnet_generic_eval_spb(*shape, int(dtype == F64))
           for k, (shape, dtype) in KERNELS.items() if k != "mnist_eval"}
    assert got == {k: 4 if k == "generic_f64_8x3x128" else 8 for k in got}
    assert ext.convnet_generic_smem_bytes(8, 3, 128, 1, 8) > ext.convnet_generic_smem_bytes(8, 3, 128, 1, 4)


@pytest.mark.parametrize("kernel", ["mnist_eval", "generic_f64_paper"])
def test_one_cta_per_node_walks_every_chunk(kernel):
    """As many nodes as SMs: the grid gives each node ``sms // L = 1`` CTA, which walks all 126 chunks of 1003
    samples (smem reused across chunks, the fc1 weight barrier past its first phase, a partial last chunk)."""
    L = torch.cuda.get_device_properties(DEV).multi_processor_count
    pr = _problem(kernel, 1003, L=L, M=8)
    _check(pr, kernel, f"L={L}")


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("train_rows,val_rows", [("f32", "u8_norm"), ("u8", "f32_raw")])
def test_validation_rows_of_another_type_and_normalisation(kernel, train_rows, val_rows):
    """The evaluation reads the validation rows' own type and normalisation, not the training shards'."""
    pr = _problem(kernel, 203, train_rows=train_rows, val_rows=val_rows)
    assert (pr.shards.x.dtype == torch.uint8) == (train_rows == "u8")
    assert (pr.val.x.dtype == torch.uint8) == (val_rows == "u8_norm")
    _check(pr, kernel, f"train {train_rows} val {val_rows}")


@pytest.mark.parametrize("kernel", ["mnist_eval", "generic_f64_paper", "generic_f32_2x5x32"])
def test_exact_logit_tie_goes_to_the_first_class(kernel):
    """Node 1's class 7 is a copy of class 3 (row of W2 and bias), both biases raised by 50: every sample's logits
    tie exactly between classes 3 and 7.  The first maximum wins, as in ``torch.argmax``: labels 3 are correct, labels
    7 are not."""
    pr = _problem(kernel, 203, val=synthetic_mnist(203, seed=4, classes=[3, 7]))
    spec = pr.base_model.spec
    (o2, s2), (ob2, _) = ko.slots(spec)[4], ko.slots(spec)[5]
    th = pr.arena.theta[1]
    w2 = th[o2: o2 + math.prod(s2)].view(s2)
    w2[7] = w2[3]
    th[ob2 + 7] = th[ob2 + 3]
    th[ob2 + 3] += 50.0
    th[ob2 + 7] += 50.0
    loss, ok = _validate(pr)
    y = pr.val.y
    assert (y == 3).any() and (y == 7).any()
    assert torch.equal(ok[1], y == 3), "a tie must go to the first class"
    nll, _ = _oracle(pr, 1)
    tol = dict(rtol=1e-9, atol=1e-11) if KERNELS[kernel][1] == F64 else dict(rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(loss[1].double(), nll, **tol)


@pytest.mark.parametrize("kernel", ["mnist_eval", "generic_f64_paper", "generic_f32_8x3x128"])
def test_evaluate_metrics_reproduce_the_oracle(kernel):
    """``validation_loss`` is the sum of batch means over ``val_batch_size`` (which does not divide V) over V,
    ``top1_accuracy`` the share of correct flags and ``true_val_loss`` the plain mean, per node."""
    V, vb = 203, 64
    pr = _problem(kernel, V, val_batch=vb)
    dtype = KERNELS[kernel][1]
    pr.evaluate_metrics()
    tol = dict(rtol=1e-9, atol=1e-12) if dtype == F64 else dict(rtol=1e-5, atol=1e-7)
    for l in range(pr.placement.L):
        nll, z = _oracle(pr, l)
        batch_means = sum(nll[i: i + vb].mean() for i in range(0, V, vb))     # the last batch holds 11 samples
        torch.testing.assert_close(pr.metrics["validation_loss"][-1][l].double(), batch_means.cpu() / V, **tol)
        torch.testing.assert_close(pr.true_val_loss[l].double(), nll.mean().cpu(), **tol)
        acc_ref = (z.argmax(1) == pr.val.y).double().mean().item()
        slack = int((_margin(z) <= (1e-9 if dtype == F64 else 1e-4)).sum()) / V
        assert abs(pr.metrics["top1_accuracy"][-1][l].item() - acc_ref) <= slack + (1e-12 if dtype == F64 else 1e-6)


@pytest.mark.parametrize("kernel", ["mnist_eval", "generic_f64_paper", "generic_f32_2x5x32"])
def test_validate_between_training_steps_changes_nothing(kernel):
    """Two training steps with a ``validate()`` between them leave ``arena.grad``, the draw counters and the losses
    bit-identical to two steps without it: evaluation shares no buffer with training."""
    outs = []
    for with_eval in (False, True):
        pr = _problem(kernel, 203)
        losses = [pr.compute_grads().clone()]
        if with_eval:
            _validate(pr)
        losses.append(pr.compute_grads().clone())
        torch.cuda.synchronize()
        outs.append((pr.arena.grad.clone(), pr.fused.calls.clone(), pr.calls.copy(), torch.stack(losses)))
    (g0, c0, h0, l0), (g1, c1, h1, l1) = outs
    assert torch.equal(g0, g1) and torch.equal(c0, c1) and (h0 == h1).all() and torch.equal(l0, l1)
