"""CPU checks of the fp64 oracles in ``kernel_oracles``: they compute what they claim, and the acceptance check built
on them rejects the tile-level bugs the GPU kernel tests rely on it to catch."""
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.data.mnist import MNIST_MEAN, MNIST_STD, synthetic_mnist
from nn_distributed_training_b200.models import FourierNet, MNISTConvNet
from nn_distributed_training_b200.models.relu_nn import FFReLUNet
from nn_distributed_training_b200.parallel.arena import FlatLayout

LOSSES = {"BCE": torch.nn.BCELoss, "MSE": torch.nn.MSELoss, "L1": torch.nn.L1Loss}


def _row(model):
    return ko.flatten([p.detach().to(torch.float64) for p in model.parameters()], model.spec,
                      FlatLayout.from_module(model).n_pad)


def _density_batch(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, 2, generator=g) - 0.5) * 1200
    y = (torch.rand(n, generator=g) < 0.3).float()
    return x, y


def _fourier(h1, dtype=None, seed=0):
    torch.manual_seed(seed)
    return FourierNet([2, h1, 64, 64, 64, 1], scale=0.05, dtype=dtype)


# ---- the oracles compute what they claim ----------------------------------------------------------------------------
@pytest.mark.parametrize("h1", [64, 128, 256])
@pytest.mark.parametrize("net,loss", [("fourier", "BCE"), ("fourier", "MSE"), ("fourier", "L1"),
                                      ("relu", "MSE"), ("relu", "L1")])
def test_exact_mlp_matches_fp64_autograd(net, loss, h1):
    torch.manual_seed(1)
    model = _fourier(h1, torch.float64) if net == "fourier" else FFReLUNet([2, h1, 64, 64, 64, 1], dtype=torch.float64)
    x, y = _density_batch(300)
    if net == "relu":
        x = x / 600.0
    x, y = x.double(), y.double()
    out = LOSSES[loss]()(model(x).squeeze(), y)
    ref = torch.autograd.grad(out, list(model.parameters()))
    l, g, _ = ko.mlp_bf16_faithful(_row(model), model.spec, x, y, loss, rounding=False)
    torch.testing.assert_close(l, out.detach(), rtol=1e-12, atol=0)
    for (o, s), r in zip(ko.slots(model.spec), ref):
        torch.testing.assert_close(g[o: o + r.numel()].reshape(s), r, rtol=1e-12, atol=1e-12 * r.abs().max().item())


def test_bf16_rounding_matches_torch_cast():
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(100000, generator=g) * 10.0 ** torch.randint(-20, 20, (100000,), generator=g),
                   torch.tensor([0.0, -0.0, 1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 3.0e38])])
    assert torch.equal(ko.round_bf16(x), x.to(torch.bfloat16).to(torch.float64))
    assert torch.equal(ko.round_bf16(x.double()), x.to(torch.bfloat16).to(torch.float64))


def test_tf32_rounding_hand_values():
    e = 2.0 ** -10                                     # TF32 spacing at 1
    cases = {1.0: 1.0, 1.0 + e: 1.0 + e, 1.0 + e / 4: 1.0, 1.0 + 3 * e / 4: 1.0 + e,
             1.0 + e / 2: 1.0 + e,                     # tie: away from zero
             1.0 + 3 * e / 2: 1.0 + 2 * e,             # tie: away from zero, not to even
             -(1.0 + e / 2): -(1.0 + e), 0.1: 0.0999755859375, 3.14159265: 3.140625, -1e-3: -0.0010004043579101562}
    got = ko.round_tf32(torch.tensor(list(cases), dtype=torch.float64))
    assert got.tolist() == list(cases.values())
    # and the result has at most 11 significant bits
    x = torch.randn(10000, dtype=torch.float64)
    m, _ = torch.frexp(ko.round_tf32(x))
    assert torch.equal(m * 2048, torch.round(m * 2048))


def test_convnet_oracle_matches_module_autograd():
    torch.manual_seed(0)
    model = MNISTConvNet(3, 5, 64, dtype=torch.float64)
    sh = synthetic_mnist(40, seed=5)
    x = (sh.x.double() / 255 - MNIST_MEAN) / MNIST_STD
    out = torch.nn.NLLLoss()(model(x), sh.y)
    ref = torch.autograd.grad(out, list(model.parameters()))
    l, g = ko.convnet_fp64(_row(model), model.spec, sh.x, sh.y, MNIST_MEAN, MNIST_STD)
    torch.testing.assert_close(l, out.detach(), rtol=1e-13, atol=0)
    torch.testing.assert_close(g, _row_of_tensors(ref, model), rtol=1e-12, atol=1e-15)


def test_convnet_eval_oracle_matches_module_per_sample():
    torch.manual_seed(0)
    model = MNISTConvNet(3, 5, 64, dtype=torch.float64)
    sh = synthetic_mnist(300, seed=6)
    x = (sh.x.double() / 255 - MNIST_MEAN) / MNIST_STD
    with torch.no_grad():
        out = model(x)
    ref = torch.nn.NLLLoss(reduction="none")(out, sh.y)
    nll, z = ko.convnet_fp64_eval(_row(model), model.spec, sh.x, sh.y, MNIST_MEAN, MNIST_STD)
    assert nll.shape == (300,) and z.shape == (300, 10) and nll.dtype == torch.float64
    torch.testing.assert_close(nll, ref, rtol=1e-13, atol=0)
    assert torch.equal(z.argmax(1), out.argmax(1))
    loss = ko.convnet_fp64(_row(model), model.spec, sh.x, sh.y, MNIST_MEAN, MNIST_STD)[0]
    torch.testing.assert_close(nll.mean(), loss, rtol=1e-14, atol=0)
    # float rows go in as they are, without the normalisation
    nf, _ = ko.convnet_fp64_eval(_row(model), model.spec, x.float(), sh.y)
    torch.testing.assert_close(nf, nll, rtol=1e-6, atol=1e-7)


def _pool_argmax_fp64(x, wc, bc):
    c = torch.nn.functional.conv2d((x.double() / 255 - MNIST_MEAN) / MNIST_STD, wc, bc)
    win = c.unfold(2, 2, 2).unfold(3, 2, 2).flatten(-2)
    top = win.topk(2, -1).values
    return win.argmax(-1), top[..., 0] - top[..., 1]


def test_fp32_pool_decisions_explain_the_near_tie_at_batch_100():
    """Node 0's first draw at batch 100 in the batch-split kernel test (one class per node, 151 rows) holds one
    max-pool window whose two largest conv outputs differ by less than fp32 resolves (7e-8 in fp64).  The fp32 conv of
    the kernels (``_pool_argmax_f32``) picks the other position there, and that one rerouted cell alone puts the
    conv-weight gradient at more than 0.1x the 1xTF32 yardstick's error against the fp64 routing: what
    ``pool_f32`` takes out of the comparison.  On a batch without such a window the two oracles are identical."""
    torch.manual_seed(0)
    model = MNISTConvNet(3, 5, 64)
    sh = synthetic_mnist(151, seed=100, classes=[0])
    row = _row(model)
    wc, bc = (t.double() for t in ko.unflatten(row, model.spec)[:2])
    rows = ko.batch_rows([151] * 3, 100, 7, 0, 0)
    x = sh.x[rows]
    a64, gap = _pool_argmax_fp64(x, wc, bc)
    differ = a64 != ko._pool_argmax_f32(x, wc, MNIST_MEAN, MNIST_STD)
    assert int(differ.sum()) == 1 and gap[differ].item() < 1e-7
    args = (model.spec, x, sh.y[rows], MNIST_MEAN, MNIST_STD)
    ref, yard = ko.convnet_fp64(row, *args)[1], ko.convnet_fp64(row, *args, tf32_fc1=True)[1]
    rerouted = ko.convnet_fp64(row, *args, pool_f32=True)[1]
    rat = ko.error_ratios(rerouted, ref, yard, model.spec)
    assert max(rat["p0"]) > ko.CONVNET_FRAC and max(max(v) for k, v in rat.items() if k != "p0") < ko.CONVNET_FRAC
    other = ko.batch_rows([151] * 3, 100, 7, 0, 1)
    x = sh.x[other]
    assert torch.equal(_pool_argmax_fp64(x, wc, bc)[0], ko._pool_argmax_f32(x, wc, MNIST_MEAN, MNIST_STD))
    args = (model.spec, x, sh.y[other], MNIST_MEAN, MNIST_STD)
    assert torch.equal(ko.convnet_fp64(row, *args, pool_f32=True)[1], ko.convnet_fp64(row, *args)[1])


def _eval_vectors(V=301):
    """The per-sample losses of an fp32 forward (a correct evaluation kernel), the fp64 oracle and the 1xTF32
    yardstick, as dicts of one vector each."""
    torch.manual_seed(0)
    model = MNISTConvNet(3, 5, 64)
    sh = synthetic_mnist(V, seed=7)
    row = _row(model)
    args = (model.spec, sh.x, sh.y, MNIST_MEAN, MNIST_STD)
    ref = ko.convnet_fp64_eval(row, *args)[0]
    tf32 = ko.convnet_fp64_eval(row, *args, tf32_fc1=True)[0]
    fp32 = ko.convnet_fp64_eval(row, *args, dtype=torch.float32)[0].double()
    return {"loss": fp32}, {"loss": ref}, {"loss": tf32}


def test_fp32_per_sample_losses_pass_the_convnet_check():
    got, ref, yard = _eval_vectors()
    rat = ko.assert_close_to_oracle(got, ref, yard, ko.CONVNET_FRAC, block=(128, 1))
    assert 0 < max(rat["loss"])


def test_stale_eval_chunk_is_rejected():
    """An evaluation CTA that stores one 8-sample chunk with the values of the chunk before it (smem not refreshed
    between chunks) must fail the per-sample check."""
    got, ref, yard = _eval_vectors()
    bad = got["loss"].clone()
    bad[200:208] = bad[192:200]
    with pytest.raises(AssertionError, match=f"above {ko.CONVNET_FRAC}"):
        ko.assert_close_to_oracle({"loss": bad}, ref, yard, ko.CONVNET_FRAC, block=(128, 1))


def _row_of_tensors(ts, model):
    return ko.flatten(list(ts), model.spec, FlatLayout.from_module(model).n_pad)


def test_batch_rows_follow_the_sampler_and_shard_offsets():
    from nn_distributed_training_b200.data.sampler import BatchSchedule
    sizes = [10, 7, 12]
    rows = ko.batch_rows(sizes, 4, 3, 2, 3, node0=5)      # node 2: its 4th draw is the partial batch of epoch 0
    assert rows.tolist() == (17 + BatchSchedule(12, 4).indices(3, 3, 7)).tolist()
    assert len(ko.batch_rows(sizes, 4, 3, 1, 1)) == 3
    assert sorted(torch.cat([ko.batch_rows(sizes, 4, 3, 0, c) for c in range(3)]).tolist()) == list(range(10))


# ---- the acceptance check catches the bugs it is meant to catch -------------------------------------------------------
def _mlp_case(h1=128, B=300, loss="BCE"):
    model = _fourier(h1)
    x, y = _density_batch(B, seed=2)
    row = _row(model)
    cache = {}
    ref = ko.mlp_bf16_faithful(row, model.spec, x, y, loss, cache=cache)[1]
    kern = ko.mlp_bf16_faithful(row, model.spec, x, y, loss, accum=torch.float32)[1].double()   # a correct kernel
    yard = ko.mlp_bf16_faithful(row, model.spec, x, y, loss, rounding=False)[1]
    return model, x, y, row, ref, kern, yard, cache


@pytest.mark.parametrize("h1,B,loss", [(128, 300, "BCE"), (256, 1000, "MSE"), (64, 129, "L1")])
def test_fp32_accumulation_passes_the_mlp_check(h1, B, loss):
    _, _, _, _, ref, kern, yard, _ = _mlp_case(h1, B, loss)
    rat = ko.assert_close_to_oracle(kern, ref, yard, ko.MLP_FRAC, spec=_fourier(h1).spec)
    assert max(max(v) for v in rat.values()) > 0      # fp32 accumulation is not bit-identical: the check compares


def _rejected(got, ref, yard, spec, frac=ko.MLP_FRAC):
    with pytest.raises(AssertionError, match=f"above {frac}"):
        ko.assert_close_to_oracle(got, ref, yard, frac, spec=spec)


def test_zeroed_mma_tile_of_dw1_is_rejected():
    model, _, _, _, ref, kern, yard, _ = _mlp_case()
    o, s = ko.slots(model.spec)[2]                        # W1 [64, h1]
    bad = kern.clone()
    bad[o: o + s[0] * s[1]].view(s)[16:32, 40:48] = 0.0
    _rejected(bad, ref, yard, model.spec)


def test_missing_k_step_of_dw2_is_rejected():
    model, _, _, _, ref, kern, yard, c = _mlp_case()
    o, s = ko.slots(model.spec)[4]                        # W2 [64, 64] = dz3^T h2 over the batch rows
    rows = slice(128 + 32, 128 + 48)                      # the third 16-row k-step of the second tile
    bad = kern.clone()
    bad[o: o + 4096] -= (c["dz3"][rows].T @ c["h2"][rows]).reshape(-1)
    _rejected(bad, ref, yard, model.spec)


def test_tile_stored_instead_of_added_is_rejected():
    """A CTA that walks tiles 0 and 1 of a node but stores tile 1's weight gradients over tile 0's (``acc_store`` with
    add = false): the node's gradient misses tile 0.  The fp32 w4 / b4 accumulators are not written by acc_store."""
    model, x, y, row, ref, kern, yard, _ = _mlp_case()
    tile0 = ko.mlp_bf16_faithful(row, model.spec, x[:128], y[:128], "BCE", batch_size=300)[1]
    o8 = ko.slots(model.spec)[8][0]
    bad = kern.clone()
    bad[:o8] -= tile0[:o8]
    _rejected(bad, ref, yard, model.spec)


def test_one_tf32_pass_is_rejected_and_fp32_passes_the_convnet_check():
    torch.manual_seed(0)
    model = MNISTConvNet(3, 5, 64)
    sh = synthetic_mnist(64, seed=101, classes=[1])
    row = _row(model)
    args = (model.spec, sh.x, sh.y, MNIST_MEAN, MNIST_STD)
    ref = ko.convnet_fp64(row, *args)[1]
    tf32 = ko.convnet_fp64(row, *args, tf32_fc1=True)[1]
    fp32 = ko.convnet_fp64(row, *args, dtype=torch.float32)[1].double()     # an fp32-exact kernel
    ko.assert_close_to_oracle(fp32, ref, tf32, ko.CONVNET_FRAC, spec=model.spec)
    _rejected(tf32, ref, tf32, model.spec, ko.CONVNET_FRAC)


def test_saturated_bce_rows_in_fp32_autograd():
    """What the torch backend does on a saturated BCE row, the case where the fused kernel differs: in fp32 the
    sigmoid rounds to 1, BCELoss reports its clamped -100 log, and autograd returns a zero gradient; the kernel keeps
    the same clamped loss but takes the gradient of the exact loss, p - y = 1 (tests/test_gpu_mlp.py)."""
    z = torch.tensor([30.0], requires_grad=True)
    loss = torch.nn.BCELoss()(torch.sigmoid(z), torch.tensor([0.0]))
    loss.backward()
    assert loss.item() == 100.0
    assert z.grad.item() == 0.0
    zd = torch.tensor([30.0], dtype=torch.float64)
    assert abs(torch.sigmoid(zd).item() - 1.0) < 1e-12 and torch.sigmoid(zd).item() != 1.0


def test_fp32_references_turns_tf32_off_and_restores_it():
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
    try:
        with ko.fp32_references():
            assert not torch.backends.cudnn.allow_tf32 and not torch.backends.cuda.matmul.allow_tf32
        assert torch.backends.cudnn.allow_tf32 and torch.backends.cuda.matmul.allow_tf32
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
