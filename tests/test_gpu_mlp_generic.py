"""The generic CUDA-core MLP kernels ``mlp_generic_forward_kernel<T>`` / ``mlp_generic_backward_kernel<T>``
(csrc/mlp_generic.cu) against the float64 oracle ``kernel_oracles.mlp_fp64``: the output, every saved activation,
every parameter gradient and dx.

The kernels run every ``FFReLUNet / FFTanhNet / FFSigmoidNet`` on CUDA, the RL actors and critics among them.  The
forward dispatches each layer on ``dpad = next_pow2(max(8, dout))`` to RG = dpad / 8 rows per thread; the cases put
``dout`` on both sides of every boundary (8/9, 16/17, 32/33, 64/65, 128/129, 256), ``din`` at 1, 31, 32, 33 and 256
(a partial 32-wide K chunk, one full chunk, a full and a partial one, eight full ones), one and eight layers, every activation as a hidden and as the
last layer, batches of 1 .. 50000 rows (32 per CTA), and inputs without ``requires_grad`` (the backward's
``gx == nullptr`` early exit, the RL path: observations carry no gradient).

float64 is held to rtol 1e-9; fp32 to ``TF32_POINT_FRAC`` of the error of ``mlp_fp64`` at the TF32 rounding of the
parameters, the rows and dL/dout, per tensor and per 16 x 8 block."""
import math

import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.ops import load_ext
from nn_distributed_training_b200.ops import mlp_generic as mg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32, F64 = torch.float32, torch.float64
R, T, S, N = "relu", "tanh", "sigmoid", "none"

# id -> (shape, activations, leading dims of x, x.requires_grad)
CASES = {
    "douts_8_to_65": ([33, 8, 9, 16, 17, 32, 33, 64, 65], [R, T, S, N, R, T, S, N], (2400,), True),
    "douts_128_to_256": ([31, 128, 129, 256, 1], [T, R, N, S], (33,), True),
    "one_unit": ([1, 1], [N], (1,), True),
    "din32_relu_last": ([32, 64, 17], [N, R], (31,), False),
    "din256_one_layer_tanh": ([256, 256], [T], (32,), True),
    "rl_actor_50000": ([12, 64, 64, 64, 5], [R, R, R, N], (50000,), False),
    "din33_3d_input": ([33, 20, 3], [S, T], (7, 9), True),
    "eight_layers": ([256, 9, 17, 33, 65, 129, 256, 8, 1], [R, T, S, N, R, T, S, N], (300,), True),
}


def _dpad(dout):
    return max(8, 1 << (int(dout) - 1).bit_length())


def _inputs(shape, lead, dtype, seed=0):
    """``nn.Linear``-style parameters in the flat layout, rows ``x [*lead, d0]`` and ``dL/dout``."""
    g = torch.Generator().manual_seed(seed)
    flat = ko.mlp_params(shape, seed).to(dtype).to(DEV)
    x = torch.randn(*lead, shape[0], generator=g).to(dtype).to(DEV)
    gout = torch.randn(*lead, shape[-1], generator=g).to(dtype).to(DEV)
    return flat, x, gout


def _oracle(flat, shape, acts, x, gout, with_acts=True, with_dx=True):
    """The fp64 oracle and its TF32-point yardstick as dicts of tensors."""
    x2, g2 = x.reshape(-1, shape[0]), gout.reshape(-1, shape[-1])
    out = []
    for f, xx, gg in ((flat, x2, g2), (ko.round_tf32(flat), ko.round_tf32(x2), ko.round_tf32(g2))):
        o, hs, gp, dx = ko.mlp_fp64(f, shape, acts, xx, gg)
        out.append(ko.mlp_named(shape, o, hs if with_acts else None, gp, dx if with_dx else None))
    return out


def _check(got, ref, yard, dtype, tag):
    if dtype == F64:
        worst = 0.0
        for k, r in ref.items():
            atol = 1e-11 * max(1.0, r.abs().max().item())
            torch.testing.assert_close(got[k].double(), r, rtol=1e-9, atol=atol, msg=lambda m: f"{k}: {m}")
            worst = max(worst, ((got[k].double() - r).abs() / (atol + 1e-9 * r.abs())).max().item())
        print(f"\nRATIO mlp_generic<double> {tag}: worst error {worst:.2e} of the tolerance")
    else:
        rat = ko.assert_close_to_oracle({k: v.double() for k, v in got.items()}, ref, yard, ko.TF32_POINT_FRAC)
        print(f"\nRATIO mlp_generic<float> {tag}: " + " ".join(f"{k}={max(v):.2e}" for k, v in rat.items()))


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", list(CASES))
def test_generic_mlp_kernels_match_fp64_oracle(case, dtype):
    """The two launches through the extension, so the saved activations are checked too.  The activation buffer and
    dx start as NaN: every entry must be written."""
    shape, acts, lead, needs_gx = CASES[case]
    flat, x, gout = _inputs(shape, lead, dtype)
    x2, g2 = x.reshape(-1, shape[0]).contiguous(), gout.reshape(-1, shape[-1]).contiguous()
    M = x2.shape[0]
    ext = load_ext(required=True)
    d, n = mg._desc(shape, acts, dtype)
    assert n == flat.numel()
    buf = torch.full((M, sum(shape[1:])), float("nan"), dtype=dtype, device=DEV)
    d.update(x=x2.data_ptr(), params=flat.data_ptr(), M=M, acts=buf.data_ptr())
    ext.mlp_generic_forward(d)
    gflat = torch.zeros_like(flat)
    gx = torch.full_like(x2, float("nan")) if needs_gx else None
    d.update(gout=g2.data_ptr(), gparams=gflat.data_ptr(), gx=None if gx is None else gx.data_ptr())
    ext.mlp_generic_backward(d)
    torch.cuda.synchronize()
    assert torch.isfinite(buf).all(), "unwritten activations"
    ends = [sum(shape[1: l + 2]) for l in range(len(shape) - 1)]
    hs = [buf[:, e - shape[l + 1]: e] for l, e in enumerate(ends)]
    got = ko.mlp_named(shape, hs[-1], hs, gflat, gx)
    ref, yard = _oracle(flat, shape, acts, x2, g2, with_dx=needs_gx)
    _check(got, ref, yard, dtype, f"{case} M={M}")


MODULES = {"FFReLUNet": ([12, 64, 64, 64, 5], (4, 600)), "FFTanhNet": ([2, 37, 129, 3], (100,)),
           "FFSigmoidNet": ([7, 256, 16, 8], (5, 13))}


@pytest.mark.parametrize("needs_gx", [True, False], ids=["x_grad", "no_x_grad"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("cls_name", list(MODULES))
def test_ffnet_forward_runs_the_kernels_and_matches_fp64_oracle(cls_name, dtype, needs_gx, monkeypatch):
    """``FFxNet.forward`` on CUDA (the fused autograd function): output, every parameter's ``.grad`` and ``x.grad``,
    on inputs with leading dimensions (``[T, E, d0]`` for two of them)."""
    from nn_distributed_training_b200.models import relu_nn
    monkeypatch.delenv("NNDT_FUSED_MLP", raising=False)
    shape, lead = MODULES[cls_name]
    net = getattr(relu_nn, cls_name)(shape, dtype=dtype).to(DEV)
    acts = net._layer_acts()
    flat, x, gout = _inputs(shape, lead, dtype, seed=1)
    with torch.no_grad():
        torch.nn.utils.vector_to_parameters(flat, net.parameters())
    x.requires_grad_(needs_gx)
    called = []
    real = mg.fused_mlp
    monkeypatch.setattr(mg, "fused_mlp", lambda *a: called.append(1) or real(*a))
    out = net(x)
    assert called, "FFxNet.forward did not run the fused kernels"
    assert out.shape == (*lead, shape[-1])
    (out * gout).sum().backward()
    gflat = torch.cat([p.grad.reshape(-1) for p in net.parameters()])
    got = ko.mlp_named(shape, out.detach(), None, gflat, x.grad if needs_gx else None)
    ref, yard = _oracle(flat, shape, acts, x.detach(), gout, with_acts=False, with_dx=needs_gx)
    _check(got, ref, yard, dtype, f"{cls_name} x{list(x.shape)}")


def test_cases_run_every_dispatch_class():
    """Every case runs in both dtypes, so the table covers all 12 ``(dtype, dpad)`` forward classes, and at least
    one case leaves dx out (the backward's ``gx == nullptr`` exit)."""
    dpads = {_dpad(d) for shape, _, _, _ in CASES.values() for d in shape[1:]}
    assert {(t, p) for t in (F32, F64) for p in dpads} == {(t, 8 << i) for t in (F32, F64) for i in range(6)}
    assert any(not needs_gx for *_, needs_gx in CASES.values())
    assert {1, 8} <= {len(shape) - 1 for shape, *_ in CASES.values()}
    assert {1, 31, 32, 33, 256} <= {shape[0] for shape, *_ in CASES.values()}
    assert {1, 31, 32, 33, 2400, 50000} <= {math.prod(lead) for _, _, lead, _ in CASES.values()}
    last = {acts[-1] for _, acts, _, _ in CASES.values()}
    hidden = {a for _, acts, _, _ in CASES.values() for a in acts[:-1]}
    assert last == hidden == {R, T, S, N}


@pytest.mark.parametrize("what", ["f64_params_f32_x", "f32_params_f64_x", "narrow_x", "wide_x"])
def test_mismatched_arguments_raise_what_sequential_raises(what, monkeypatch):
    """Parameters of another dtype than x, or x of another width than ``shape[0]``: the fused path must not read
    them as raw arrays (garbage, or out of bounds) but raise the error ``nn.Sequential`` raises."""
    from nn_distributed_training_b200.models.relu_nn import FFReLUNet
    shape = [12, 64, 5]
    pdt, xdt, width = {"f64_params_f32_x": (F64, F32, 12), "f32_params_f64_x": (F32, F64, 12),
                       "narrow_x": (F32, F32, 11), "wide_x": (F32, F32, 13)}[what]
    net = FFReLUNet(shape, dtype=pdt).to(DEV)
    x = torch.randn(40, width, dtype=xdt, device=DEV)
    errors = []
    for fused in ("1", "0"):
        monkeypatch.setenv("NNDT_FUSED_MLP", fused)
        with pytest.raises(RuntimeError) as e:
            net(x)
        errors.append(type(e.value))
    torch.cuda.synchronize()
    assert errors[0] is errors[1]
