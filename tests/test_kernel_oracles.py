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


# ---- the generic CUDA-core conv-net kernel: oracle, TF32-point yardstick, mutations ----------------------------------
GENERIC_SHAPES = [(1, 3, 1), (1, 5, 10), (8, 5, 128), (2, 3, 33), (3, 5, 64)]


@pytest.mark.parametrize("shape", [(1, 3, 1), (8, 5, 128)])
def test_convnet_oracle_matches_module_autograd_at_generic_edges(shape):
    torch.manual_seed(0)
    model = MNISTConvNet(*shape, dtype=torch.float64)
    sh = synthetic_mnist(37, seed=5)
    x = (sh.x.double() / 255 - MNIST_MEAN) / MNIST_STD
    out = torch.nn.NLLLoss()(model(x), sh.y)
    ref = torch.autograd.grad(out, list(model.parameters()))
    l, g = ko.convnet_fp64(_row(model), model.spec, sh.x, sh.y, MNIST_MEAN, MNIST_STD)
    torch.testing.assert_close(l, out.detach(), rtol=1e-13, atol=0)
    torch.testing.assert_close(g, _row_of_tensors(ref, model), rtol=1e-12, atol=1e-15)


def _generic_conv_case(shape, B, float_rows=False, draw=0):
    """One node of the generic-kernel GPU test on CPU: its rows for ``draw`` (0: a full batch, 1: the partial one),
    the fp64 oracle, the TF32-point yardstick and fp32 autograd standing in for an fp32-exact kernel."""
    torch.manual_seed(0)
    model = MNISTConvNet(*shape)
    M = B + B // 2 + 1
    sh = synthetic_mnist(M, seed=100, classes=[0])
    rows = ko.batch_rows([M], B, 7, 0, draw)
    x, y = sh.x[rows], sh.y[rows]
    mean, std = MNIST_MEAN, MNIST_STD
    if float_rows:
        x, mean, std = ((x.double() / 255 - MNIST_MEAN) / MNIST_STD).float(), 0.0, 1.0
    row = _row(model)
    o, (lw,) = ko.slots(model.spec)[3]
    row[o: o + lw] = row[o: o + lw].abs() + 0.1           # b1 > 0: at linear width 1 a dead unit zeroes every gradient
    args = (model.spec, x, y, mean, std)
    ref = ko.convnet_fp64(row, *args, pool_f32=True)[1]
    yard = ko.convnet_tf32_point(row, *args)[1]
    fp32 = ko.convnet_fp64(row, *args, dtype=torch.float32)[1].double()
    return model, row, args, ref, yard, fp32


@pytest.mark.parametrize("float_rows", [False, True], ids=["u8", "f32"])
@pytest.mark.parametrize("B", [8, 37])
@pytest.mark.parametrize("shape", GENERIC_SHAPES)
def test_fp32_autograd_passes_the_tf32_point_convnet_check(shape, B, float_rows):
    for draw in (0, 1):
        model, _, _, ref, yard, fp32 = _generic_conv_case(shape, B, float_rows, draw)
        assert all(t.abs().max() > 0 for t in ko.unflatten(ref, model.spec))
        rat = ko.assert_close_to_oracle(fp32, ref, yard, ko.TF32_POINT_FRAC, spec=model.spec)
        print(f"\nRATIO {shape} B={B} draw {draw}: " + " ".join(f"{k}={max(v):.2e}" for k, v in rat.items()))


def test_partial_batch_divided_by_the_batch_size_is_rejected():
    """The partial batch (19 of 37 rows) scaled by 1 / 37 instead of 1 / 19, and by 1 / 20."""
    model, _, args, ref, yard, fp32 = _generic_conv_case((2, 3, 33), 37, draw=1)
    n = args[1].shape[0]
    assert n == 19
    for wrong in (37, n + 1):
        _rejected(fp32 * n / wrong, ref, yard, model.spec, ko.TF32_POINT_FRAC)


def test_dropped_sample_of_a_slice_is_rejected():
    """A slice that skips its third sample but still divides by the batch size."""
    model, row, (spec, x, y, mean, std), ref, yard, _ = _generic_conv_case((1, 5, 10), 37)
    keep = torch.arange(x.shape[0]) != 2
    bad = ko.convnet_fp64(row, spec, x[keep], y[keep], mean, std, dtype=torch.float32)[1].double()
    _rejected(bad * (x.shape[0] - 1) / x.shape[0], ref, yard, spec, ko.TF32_POINT_FRAC)


def _conv_partition_grads(row, spec, x, y, mean, std, q, npart):
    """Conv weight and bias gradients routed through the pool cells of conv-gradient partition ``q`` of ``npart``
    (cells ``q NP / npart .. (q + 1) NP / npart - 1`` of every filter, as ``generic_chunk`` splits them)."""
    wc, bc, w1, b1, w2, b2 = params = [p.requires_grad_(True) for p in ko.unflatten(row, spec)]
    xin = (x.double().reshape(-1, 1, 28, 28) / 255.0 - mean) / std
    a = torch.nn.functional.max_pool2d(torch.relu(torch.nn.functional.conv2d(xin, wc, bc)), 2)
    npos = a.shape[-1] ** 2
    p = torch.arange(npos)
    keep = ((p >= q * npos // npart) & (p < (q + 1) * npos // npart)).double().reshape(a.shape[-2:])
    a.register_hook(lambda g: g * keep)
    z = torch.relu(a.flatten(1) @ w1.T + b1) @ w2.T + b2
    loss = torch.nn.functional.nll_loss(torch.log_softmax(z, 1), y)
    return torch.autograd.grad(loss, [wc, bc])


@pytest.mark.parametrize("shape,npart", [((8, 5, 128), 2), ((1, 3, 1), 51)])
def test_dropped_conv_gradient_partition_is_rejected(shape, npart):
    """``npart = 512 / (F KS^2 + F)`` partitions of the pool cells: a CTA that leaves one partition's partial out of
    the conv weight and bias gradients."""
    F_, KS = shape[:2]
    assert max(1, 512 // (F_ * KS * KS + F_)) == npart
    model, row, args, ref, yard, fp32 = _generic_conv_case(shape, 37)
    gwc, gbc = _conv_partition_grads(row, *args, q=npart // 2, npart=npart)
    (owc, swc), (obc, _) = ko.slots(model.spec)[:2]
    bad = fp32.clone()
    bad[owc: owc + gwc.numel()] -= gwc.reshape(-1)
    bad[obc: obc + gbc.numel()] -= gbc
    _rejected(bad, ref, yard, model.spec, ko.TF32_POINT_FRAC)


# ---- the generic CUDA-core MLP kernels: oracle, TF32-point yardstick, mutations --------------------------------------
ACT_MIXES = [([5, 7, 3], ["relu", "none"]), ([5, 7, 3], ["tanh", "tanh"]), ([5, 7, 3], ["sigmoid", "sigmoid"]),
             ([4, 9, 6, 8, 2], ["none", "relu", "tanh", "sigmoid"]), ([3, 6, 6, 4], ["sigmoid", "none", "relu"]),
             ([2, 5, 1], ["tanh", "relu"]), ([1, 1], ["none"])]
ACT_MODULES = {"none": torch.nn.Identity, "relu": torch.nn.ReLU, "tanh": torch.nn.Tanh, "sigmoid": torch.nn.Sigmoid}


@pytest.mark.parametrize("shape,acts", ACT_MIXES)
def test_mlp_oracle_matches_sequential_autograd(shape, acts):
    flat = ko.mlp_params(shape)
    mods = []
    for l, a in enumerate(acts):
        lin = torch.nn.Linear(shape[l], shape[l + 1], dtype=torch.float64)
        wo, bo = ko.mlp_layout(shape)[l]
        with torch.no_grad():
            lin.weight.copy_(flat[wo: bo].reshape(lin.weight.shape))
            lin.bias.copy_(flat[bo: bo + shape[l + 1]])
        mods += [lin, ACT_MODULES[a]()]
    seq = torch.nn.Sequential(*mods)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(50, shape[0], generator=g, dtype=torch.float64, requires_grad=True)
    gout = torch.randn(50, shape[-1], generator=g, dtype=torch.float64)
    out = seq(x)
    grads = torch.autograd.grad((out * gout).sum(), [x, *seq.parameters()])
    o, hs, gflat, dx = ko.mlp_fp64(flat, shape, acts, x.detach(), gout)
    torch.testing.assert_close(o, out.detach(), rtol=1e-14, atol=1e-15)
    h = x.detach()
    for l in range(len(acts)):
        h = seq[2 * l + 1](seq[2 * l](h))
        torch.testing.assert_close(hs[l], h.detach(), rtol=1e-14, atol=1e-15)
    torch.testing.assert_close(gflat, torch.cat([t.reshape(-1) for t in grads[1:]]), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(dx, grads[0], rtol=1e-12, atol=1e-14)


class _TanhFromPreactivation(torch.autograd.Function):
    """tanh with the derivative a buggy kernel would take: 1 - z^2 of the pre-activation z instead of 1 - y^2."""

    @staticmethod
    def forward(ctx, z):
        ctx.save_for_backward(z)
        return torch.tanh(z)

    @staticmethod
    def backward(ctx, g):
        z, = ctx.saved_tensors
        return g * (1 - z * z)


def _mlp_autograd(flat, shape, acts, x, gout, tanh=torch.tanh):
    """``mlp_fp64``'s results from autograd in the dtype of the arguments."""
    flat = flat.detach().requires_grad_(True)
    x = x.detach().requires_grad_(True)
    h, hs = x, []
    for l, (wo, bo) in enumerate(ko.mlp_layout(shape)):
        z = h @ flat[wo: bo].reshape(shape[l + 1], shape[l]).T + flat[bo: bo + shape[l + 1]]
        h = tanh(z) if acts[l] == "tanh" else ko._act(z, acts[l])
        hs.append(h)
    gflat, dx = torch.autograd.grad((h * gout).sum(), [flat, x])
    return h.detach(), [t.detach() for t in hs], gflat, dx


MLP_CASES = [([12, 64, 64, 64, 5], ["relu"] * 3 + ["none"], 2400), ([12, 64, 64, 64, 1], ["relu"] * 3 + ["none"], 777),
             ([2, 37, 129, 3], ["tanh"] * 3, 100), ([7, 256, 16, 8], ["sigmoid"] * 3, 65),
             ([2, 200, 1], ["relu", "none"], 33), ([1, 1], ["none"], 31),
             ([256, 9, 17, 33, 65, 129, 256, 8, 1], ["relu", "tanh", "sigmoid", "none", "relu", "tanh", "sigmoid", "none"],
              300)]


def _mlp_generic_case(shape, acts, M, seed=0):
    g = torch.Generator().manual_seed(seed)
    flat = ko.mlp_params(shape, seed).float()
    x = torch.randn(M, shape[0], generator=g)
    gout = torch.randn(M, shape[-1], generator=g)
    ref = ko.mlp_named(shape, *ko.mlp_fp64(flat, shape, acts, x, gout))
    yard = ko.mlp_named(shape, *ko.mlp_fp64(ko.round_tf32(flat), shape, acts, ko.round_tf32(x), ko.round_tf32(gout)))
    return flat, x, gout, ref, yard


@pytest.mark.parametrize("shape,acts,M", MLP_CASES)
def test_fp32_autograd_passes_the_tf32_point_mlp_check(shape, acts, M):
    flat, x, gout, ref, yard = _mlp_generic_case(shape, acts, M)
    got = ko.mlp_named(shape, *_mlp_autograd(flat, shape, acts, x, gout))
    rat = ko.assert_close_to_oracle(got, ref, yard, ko.TF32_POINT_FRAC)
    assert 0 < max(max(v) for v in rat.values())


def _mlp_rejected(got, ref, yard):
    with pytest.raises(AssertionError, match=f"above {ko.TF32_POINT_FRAC}"):
        ko.assert_close_to_oracle(got, ref, yard, ko.TF32_POINT_FRAC)


def test_mlp_cta_missing_from_a_weight_gradient_is_rejected():
    """The RL actor at M = 2400 (75 CTAs of 32 rows): CTA 40's rows left out of W0's gradient."""
    shape, acts, M = MLP_CASES[0]
    flat, x, gout, ref, yard = _mlp_generic_case(shape, acts, M)
    got = ko.mlp_named(shape, *_mlp_autograd(flat, shape, acts, x, gout))
    rows = slice(40 * 32, 41 * 32)
    part = ko.mlp_named(shape, *ko.mlp_fp64(flat, shape, acts, x[rows], gout[rows]))
    got["W0"] = got["W0"] - part["W0"].float()
    _mlp_rejected(got, ref, yard)


def test_mlp_skipped_k_chunk_is_rejected():
    """A forward that skips the third 32-wide K chunk of the 256-wide layer 1 (``din > 32``)."""
    shape, acts, M = MLP_CASES[3]
    flat, x, gout, ref, yard = _mlp_generic_case(shape, acts, M)
    wo, bo = ko.mlp_layout(shape)[1]
    bad = flat.clone()
    bad[wo: bo].view(shape[2], shape[1])[:, 64:96] = 0.0
    got = ko.mlp_named(shape, *_mlp_autograd(bad, shape, acts, x, gout))
    got = {k: got[k] for k in ("out", "a1", "a2")}
    _mlp_rejected(got, {k: ref[k] for k in got}, {k: yard[k] for k in got})


def test_tanh_derivative_of_the_preactivation_is_rejected():
    shape, acts, M = MLP_CASES[2]
    flat, x, gout, ref, yard = _mlp_generic_case(shape, acts, M)
    got = ko.mlp_named(shape, *_mlp_autograd(flat, shape, acts, x, gout, tanh=_TanhFromPreactivation.apply))
    _mlp_rejected(got, ref, yard)


# ---- the fused MLP runs only on arguments it can read ----------------------------------------------------------------
def test_fused_mlp_arguments_must_match_dtype_device_and_width():
    from nn_distributed_training_b200.ops.mlp_generic import arguments_match
    shape = [12, 64, 5]
    params = [torch.zeros(64, 12), torch.zeros(64), torch.zeros(5, 64), torch.zeros(5)]
    assert arguments_match(torch.zeros(30, 12), params, shape)
    assert arguments_match(torch.zeros(4, 30, 12), params, shape)             # leading dims are rows
    assert not arguments_match(torch.zeros(30, 12, dtype=torch.float64), params, shape)
    assert not arguments_match(torch.zeros(30, 12), params[:3] + [torch.zeros(5, dtype=torch.float64)], shape)
    assert not arguments_match(torch.zeros(30, 11), params, shape)
    assert not arguments_match(torch.zeros(30, 13), params, shape)
    assert not arguments_match(torch.zeros(30, 12), params[:1] + [torch.zeros(64, device="meta")] + params[2:], shape)
