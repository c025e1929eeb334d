"""fp64 oracles of the tensor-core training kernels and the acceptance check that compares a kernel with them.

* ``batch_rows`` rebuilds the rows a fused kernel drew for ``(node, call)`` from the Python sampler, so an oracle runs
  on exactly the rows the kernel used without a second problem object drawing them.
* ``convnet_fp64`` is ``MNISTConvNet`` in float64 autograd (``csrc/mnist_tc.cu`` and ``csrc/mnist_cl64.cu``); with
  ``tf32_fc1=True`` the operands of its three fc1-sized contractions are rounded to TF32 first, which is the error a
  1xTF32 kernel would make: the yardstick of the 3xTF32 kernel.  ``convnet_fp64_eval`` is the same forward per sample
  (NLL and logits), the oracle of the evaluation kernels.  ``convnet_tf32_point`` is the yardstick of the fp32
  CUDA-core kernel: the oracle at the TF32 rounding of every parameter and of float rows.
* ``mlp_fp64`` is the generic feed-forward net of ``csrc/mlp_generic.cu`` (forward, saved activations, backward) in
  float64; its yardstick is the same function at the TF32 rounding of the parameters, the rows and dL/dout.
* ``mlp_bf16_faithful`` is the density MLP of ``csrc/mlp_tc.cu`` written out by hand, rounding to bf16 exactly where
  the kernel rounds and nowhere else; ``rounding=False`` gives the exact math of the same network.
* ``Guarded`` packs a kernel's output tensors, poisoned with NaN, between guard values in one buffer, so a skipped
  or an out-of-range write shows.
* ``assert_close_to_oracle`` accepts a kernel when its error is a small fraction of a yardstick's error, per tensor and
  per 16 x 8 block, so one bad MMA tile cannot hide inside a good norm.
"""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

from nn_distributed_training_b200.data.sampler import BatchSchedule
from nn_distributed_training_b200.parallel.arena import SLOT_ALIGN_ELEMS


@contextlib.contextmanager
def fp32_references():
    """fp32 autograd references run at fp32, not TF32: cuDNN convolutions allow TF32 by default, which would make a
    3xTF32 kernel look wrong against a less accurate "reference".  The previous settings are restored on exit."""
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---- rounding ------------------------------------------------------------------------------------------------------
def round_bf16(x: torch.Tensor) -> torch.Tensor:
    """Round to bfloat16 (nearest, ties to even) through the fp32 value, as ``__floats2bfloat162_rn`` does; float64
    out."""
    b = x.to(torch.float32).contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return _bits_to_f64(b)


def round_tf32(x: torch.Tensor) -> torch.Tensor:
    """Round to TF32 (10-bit mantissa, nearest, ties away from zero) through the fp32 value, as ``cvt.rna.tf32.f32``
    does; float64 out."""
    b = x.to(torch.float32).contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0x1000) & 0xFFFFE000
    return _bits_to_f64(b)


_INV_2PI_F32 = float(torch.tensor(1 / (2 * math.pi), dtype=torch.float32))


def _mul_f32_rz(a: torch.Tensor, b: float) -> torch.Tensor:
    """fp32 product of fp32 values, rounded toward zero (``FMUL.RZ``); float64 out.  The float64 product is exact."""
    p = a.to(torch.float64) * b
    r = p.to(torch.float32)
    r = torch.where(r.double().abs() > p.abs(), torch.nextafter(r, torch.zeros_like(r)), r)
    return r.to(torch.float64)


def _bits_to_f64(b: torch.Tensor) -> torch.Tensor:
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b)
    return b.to(torch.int32).view(torch.float32).to(torch.float64)


# ---- layouts and batches -------------------------------------------------------------------------------------------
def slots(spec):
    """``[(offset, shape)]`` of every parameter tensor in a node's arena row (``FlatLayout.from_module`` order)."""
    out, off = [], 0
    for shape in spec.param_shapes():
        out.append((off, tuple(shape)))
        off += -(-math.prod(shape) // SLOT_ALIGN_ELEMS) * SLOT_ALIGN_ELEMS
    return out


def unflatten(row: torch.Tensor, spec, dtype=torch.float64):
    return [row[o: o + math.prod(s)].reshape(s).to(dtype) for o, s in slots(spec)]


def flatten(tensors, spec, n_pad: int) -> torch.Tensor:
    out = torch.zeros(n_pad, dtype=tensors[0].dtype, device=tensors[0].device)
    for (o, s), t in zip(slots(spec), tensors):
        out[o: o + math.prod(s)] = t.reshape(-1)
    return out


def poison_partials(fz, spec):
    """NaN in every parameter slot of every slice's partial row of a ``FusedMnist`` and in every loss partial; the
    arena padding between the slots stays as it is (zero: the training kernels never write it)."""
    for o, s in slots(spec):
        fz.grad_part[:, :, o: o + math.prod(s)] = float("nan")
    fz.loss_part.fill_(float("nan"))


def padding_mask(spec, n_pad, device):
    """True on the arena padding of a row: the entries between (and after) the parameter slots."""
    pad = torch.ones(n_pad, dtype=torch.bool, device=device)
    for o, s in slots(spec):
        pad[o: o + math.prod(s)] = False
    return pad


def batch_rows(shard_sizes, batch: int, seed: int, node: int, call: int, node0: int = 0) -> torch.Tensor:
    """Rows of the concatenated local shards that local node ``node`` draws at its ``call``-th draw: the Feistel
    schedule of ``data.sampler`` keyed by the global node id, plus the node's shard offset."""
    off = sum(int(m) for m in shard_sizes[:node])
    return off + BatchSchedule(int(shard_sizes[node]), batch).indices(call, seed, node0 + node)


# ---- MNISTConvNet ---------------------------------------------------------------------------------------------------
class _Tf32Linear(torch.autograd.Function):
    """``a @ w.T`` with the operands of the forward and of both backward contractions rounded to TF32."""

    @staticmethod
    def forward(ctx, a, w):
        ctx.save_for_backward(a, w)
        return round_tf32(a) @ round_tf32(w).T

    @staticmethod
    def backward(ctx, g):
        a, w = ctx.saved_tensors
        gt = round_tf32(g)
        return gt @ round_tf32(w), gt.T @ round_tf32(a)


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float32).to(torch.float64)


def _pool_argmax_f32(x, wc, mean, std):
    """Argmax ``[n, F, 12, 12]`` of every 2 x 2 max-pool window as an fp32 kernel finds it: the inputs normalised in
    fp32, each conv output an ``fmaf`` chain over the taps in (ky, kx) order, the bias added after the max, and the
    first maximum winning.  (The fp64 product of two fp32 values is exact; the sum is rounded twice, which can move
    the rare ulp.)"""
    n, ks = x.shape[0], wc.shape[-1]
    if x.dtype == torch.uint8:
        xin = _f32(_f32(x.to(torch.float64) * _f32(torch.tensor(1 / 255.0)).item() - _f32(torch.tensor(mean)).item())
                   * _f32(torch.tensor(1.0 / std)).item())
    else:
        xin = _f32(x.to(torch.float64))
    xin = xin.reshape(n, 1, 28, 28)
    w = _f32(wc.detach().to(torch.float64))
    co = 28 - ks + 1
    acc = torch.zeros(n, w.shape[0], co, co, dtype=torch.float64, device=x.device)
    for ky in range(ks):
        for kx in range(ks):
            acc = _f32(w[:, 0, ky, kx].reshape(1, -1, 1, 1) * xin[:, :, ky: ky + co, kx: kx + co] + acc)
    win = acc[..., : co // 2 * 2, : co // 2 * 2].unfold(2, 2, 2).unfold(3, 2, 2).flatten(-2)
    return win.argmax(-1)                                  # the first of equal maxima, like the kernels


def _convnet_forward(params, spec, x, y, mean, std, tf32_fc1, dtype, pool_f32=False):
    """Logits ``[n, 10]`` and per-sample NLL ``[n]`` of ``MNISTConvNet`` with parameter tensors ``params`` on rows
    ``x`` (uint8 pixels normalised as ``(x / 255 - mean) / std``, or float inputs), in ``dtype``.  ``pool_f32=True``
    takes each max-pool window's argmax from ``_pool_argmax_f32`` instead: where two conv outputs of a window are
    closer than fp32 can resolve, an fp32 kernel routes that cell to another position than fp64 does."""
    wc, bc, w1, b1, w2, b2 = params
    x = x.reshape(x.shape[0], 1, spec.in_hw, spec.in_hw)
    xin = (x.to(dtype) / 255.0 - mean) / std if x.dtype == torch.uint8 else x.to(dtype)
    c = F.relu(F.conv2d(xin, wc, bc))
    if pool_f32:
        po = c.shape[-1] // 2
        win = c[..., : 2 * po, : 2 * po].unfold(2, 2, 2).unfold(3, 2, 2).flatten(-2)
        a = win.gather(-1, _pool_argmax_f32(x, wc, mean, std).unsqueeze(-1)).flatten(1)
    else:
        a = F.max_pool2d(c, 2).flatten(1)
    h = (_Tf32Linear.apply(a, w1) if tf32_fc1 else a @ w1.T) + b1
    z = F.relu(h) @ w2.T + b2
    return z, F.nll_loss(F.log_softmax(z, dim=1), y.to(z.device).long(), reduction="none")


def convnet_fp64(theta_row, spec, x, y, mean=0.0, std=1.0, tf32_fc1=False, dtype=torch.float64, pool_f32=False):
    """Mean NLL loss and flat gradient (arena layout, length of ``theta_row``) of ``MNISTConvNet`` on rows ``x``
    (uint8 pixels normalised as ``(x / 255 - mean) / std``, or float inputs), computed in ``dtype`` autograd;
    ``pool_f32``: see ``_convnet_forward``."""
    params = [p.requires_grad_(True) for p in unflatten(theta_row, spec, dtype)]
    loss = _convnet_forward(params, spec, x, y, mean, std, tf32_fc1, dtype, pool_f32)[1].mean()
    grads = torch.autograd.grad(loss, params)
    return loss.detach(), flatten([g.detach() for g in grads], spec, theta_row.shape[-1])


def convnet_tf32_point(theta_row, spec, x, y, mean=0.0, std=1.0):
    """Yardstick of the fp32 CUDA-core kernel ``convnet_generic_kernel<float, ...>``: ``convnet_fp64`` (with
    ``pool_f32``) at the TF32 rounding of every parameter and of float rows.  ``tf32_fc1`` rounds only the fc1
    contractions, so it leaves the fc2 and b2 gradients of a small net nearly exact (exact where every fc1 unit is
    off), which no fp32 kernel can match; rounding every tensor perturbs every gradient."""
    xr = x if x.dtype == torch.uint8 else round_tf32(x)
    return convnet_fp64(round_tf32(theta_row), spec, xr, y, mean, std, pool_f32=True)


def convnet_fp64_eval(theta_row, spec, x, y, mean=0.0, std=1.0, tf32_fc1=False, dtype=torch.float64):
    """Per-sample NLL ``[n]`` and logits ``[n, 10]`` of ``MNISTConvNet`` on rows ``x``, the forward of
    ``convnet_fp64``: what the evaluation kernels store per validation sample."""
    with torch.no_grad():
        z, nll = _convnet_forward(unflatten(theta_row, spec, dtype), spec, x, y, mean, std, tf32_fc1, dtype)
    return nll, z


# ---- density MLP (FourierNet / FFReLUNet [2, h1, 64, 64, 64, 1]) -----------------------------------------------------
def mlp_bf16_faithful(theta_row, spec, x, y, loss, rounding=True, accum=torch.float64, batch_size=None, cache=None):
    """Forward and backward of the density MLP written out by hand.

    ``rounding=True`` rounds to bf16 exactly where ``csrc/mlp_tc.cu`` does: W1..W3 (``stage_weight``); h1, h2, h3
    (``first_layer``, ``hidden_epilogue``); dz4, dz3, dz2 and dz1; the ``[x, 1]`` operand of the bias and first-layer
    gradients.  w0, every bias, w4, h4, the output and the loss stay unrounded; the ReLU masks of dz3 / dz2 come from
    the bf16 h, the activation derivative of dz1 from the unrounded first-layer pre-activation.  ``rounding=False`` is
    exact math of the same network and loss (BCE's logs clamped at -100 as in ``torch.nn.BCELoss``).  ``accum`` is
    the dtype every contraction and elementwise step runs in.  Gradients are divided by ``batch_size`` (default: the
    rows given).  Returns ``(loss, flat gradient, outputs p)``; ``cache`` (a dict) receives the backward operands."""
    dt = accum
    r = round_bf16 if rounding else (lambda t: t)
    rd = lambda t: r(t).to(dt)                                               # noqa: E731
    w0, b0, w1, b1, w2, b2, w3, b3, w4, b4 = unflatten(theta_row, spec, dt)
    x, y = x.to(dt), y.to(dt)
    bs = float(x.shape[0] if batch_size is None else batch_size)
    W1, W2, W3 = rd(w1), rd(w2), rd(w3)
    if rounding:
        # the first layer as the kernel evaluates it in fp32: z by two fmaf, the SFU sine of scale * z after its
        # fp32 argument reduction (multiply by 1 / 2pi, rounded toward zero).  A one-ulp change of the sine's argument
        # moves about 1e-3 of the bf16 roundings of h1, which would otherwise dominate the comparison.
        f32 = lambda t: t.to(torch.float32).to(torch.float64)               # noqa: E731
        z1 = f32(x[:, 1:2].double() * w0[:, 1].double() + f32(x[:, :1].double() * w0[:, 0].double() + b0.double()))
        turns = _mul_f32_rz(f32(spec.scale * z1), _INV_2PI_F32)
        s, c = torch.sin(2 * math.pi * turns).to(dt), torch.cos(2 * math.pi * turns).to(dt)
        z1 = z1.to(dt)
    else:
        z1 = x @ w0.T + b0
        s, c = torch.sin(spec.scale * z1), torch.cos(spec.scale * z1)
    if spec.first == "sin_relu":
        h1 = rd(torch.relu(s))
        dact1 = torch.where(s > 0, c * spec.scale, torch.zeros_like(s))
    else:
        h1 = rd(torch.relu(z1))
        dact1 = (z1 > 0).to(dt)
    h2 = rd(torch.relu(h1 @ W1.T + b1))
    h3 = rd(torch.relu(h2 @ W2.T + b2))
    h4 = torch.relu(h3 @ W3.T + b3)
    z5 = h4 @ w4.reshape(-1) + b4
    p = torch.sigmoid(z5) if spec.last == "sigmoid" else z5
    if loss == "BCE":
        lrow = -(y * torch.log(p).clamp_min(-100.0) + (1 - y) * torch.log(1 - p).clamp_min(-100.0))
        gz = (p - y) if spec.last == "sigmoid" else (p - y) / (p * (1 - p)).clamp_min(1e-12)
    else:
        dpdz = p * (1 - p) if spec.last == "sigmoid" else torch.ones_like(p)
        if loss == "MSE":
            lrow, gz = (p - y) ** 2, 2 * (p - y) * dpdz
        else:
            lrow, gz = (p - y).abs(), torch.sign(p - y) * dpdz
    d5 = gz / bs
    g_w4, g_b4 = (d5 @ h4).reshape(1, -1), d5.sum().reshape(1)
    xa = rd(torch.cat([x, torch.ones_like(x[:, :1])], 1))                   # the [x, 1] operand
    dz4 = rd(d5[:, None] * w4.reshape(1, -1) * (h4 > 0))
    g_w3, g_b3 = dz4.T @ h3, dz4.T @ xa[:, -1]
    dz3 = rd((dz4 @ W3) * (h3 > 0))
    g_w2, g_b2 = dz3.T @ h2, dz3.T @ xa[:, -1]
    dz2 = rd((dz3 @ W2) * (h2 > 0))
    g_w1, g_b1 = dz2.T @ h1, dz2.T @ xa[:, -1]
    dz1 = rd((dz2 @ W1) * dact1)
    g01 = dz1.T @ xa
    g_w0, g_b0 = g01[:, :-1], g01[:, -1]
    if cache is not None:
        cache.update(h1=h1, h2=h2, h3=h3, dz2=dz2, dz3=dz3, dz4=dz4, xa=xa)
    grads = [g_w0, g_b0, g_w1, g_b1, g_w2, g_b2, g_w3, g_b3, g_w4, g_b4]
    return lrow.sum() / bs, flatten(grads, spec, theta_row.shape[-1]), p


# ---- generic feed-forward net (FFReLUNet / FFTanhNet / FFSigmoidNet, csrc/mlp_generic.cu) -----------------------------
def mlp_layout(shape):
    """``[(w_off, b_off)]`` of every layer in the flat parameter vector of ``ops/mlp_generic.py``: W0, b0, W1, b1, ...
    back to back in ``nn.Linear`` layout."""
    out, off = [], 0
    for l in range(len(shape) - 1):
        out.append((off, off + shape[l + 1] * shape[l]))
        off += shape[l + 1] * (shape[l] + 1)
    return out


def mlp_params(shape, seed=0):
    """Flat float64 parameters of ``shape`` in the ``mlp_layout``, drawn like ``nn.Linear``'s defaults:
    U(-1 / sqrt(d_in), 1 / sqrt(d_in))."""
    g = torch.Generator().manual_seed(seed)
    ps = []
    for l in range(len(shape) - 1):
        bound = shape[l] ** -0.5
        ps += [(torch.rand(shape[l + 1] * (shape[l] + 1), generator=g, dtype=torch.float64) * 2 - 1) * bound]
    return torch.cat(ps)


def _act(z, a):
    return {"none": lambda t: t, "relu": torch.relu, "tanh": torch.tanh, "sigmoid": torch.sigmoid}[a](z)


def _act_deriv(y, a):
    """The activation's derivative written through its output ``y``."""
    if a == "relu":
        return (y > 0).to(y.dtype)
    if a == "tanh":
        return 1 - y * y
    if a == "sigmoid":
        return y * (1 - y)
    return torch.ones_like(y)


def mlp_fp64(params, shape, acts, x, gout):
    """Forward and backward of the feed-forward net ``shape`` with activations ``acts`` (one per layer) in float64,
    written out by hand: the oracle of ``mlp_generic_forward_kernel`` / ``mlp_generic_backward_kernel``.

    ``params`` is the flat vector of ``mlp_layout``, ``x`` is ``[M, shape[0]]`` and ``gout`` is ``dL/dout``
    ``[M, shape[-1]]``.  Returns ``(out, [every layer's post-activation], flat parameter gradient, dx)``."""
    shape = [int(s) for s in shape]
    p = params.to(torch.float64)
    h = [x.to(torch.float64)]
    Ws, bs = [], []
    for l, (wo, bo) in enumerate(mlp_layout(shape)):
        Ws.append(p[wo: bo].reshape(shape[l + 1], shape[l]))
        bs.append(p[bo: bo + shape[l + 1]])
        h.append(_act(h[-1] @ Ws[-1].T + bs[-1], acts[l]))
    g = torch.zeros_like(p)
    d = gout.to(torch.float64) * _act_deriv(h[-1], acts[-1])
    for l in reversed(range(len(Ws))):
        wo, bo = mlp_layout(shape)[l]
        g[wo: bo] = (d.T @ h[l]).reshape(-1)
        g[bo: bo + shape[l + 1]] = d.sum(0)
        d = d @ Ws[l]
        if l > 0:
            d = d * _act_deriv(h[l], acts[l - 1])
    return h[-1], h[1:], g, d


def mlp_named(shape, out, hs, g, dx=None):
    """``{name: tensor}`` of what ``mlp_fp64`` returns (or a kernel computed), for ``assert_close_to_oracle``: the
    output, every layer's post-activation ``a<l>``, every weight and bias gradient ``W<l>`` / ``b<l>`` and, unless
    None, ``dx``; ``hs=None`` leaves the post-activations out."""
    out_d = {"out": out.reshape(-1, int(shape[-1]))}
    for l, (wo, bo) in enumerate(mlp_layout(shape)):
        if hs is not None:
            out_d[f"a{l}"] = hs[l].reshape(-1, int(shape[l + 1]))
        out_d[f"W{l}"] = g[wo: bo].reshape(int(shape[l + 1]), int(shape[l]))
        out_d[f"b{l}"] = g[bo: bo + int(shape[l + 1])]
    if dx is not None:
        out_d["dx"] = dx.reshape(-1, int(shape[0]))
    return out_d


# ---- poisoned outputs -----------------------------------------------------------------------------------------------
class Guarded:
    """Tensors of the given shapes, each filled with NaN, packed in one buffer with ``gap`` guard values before,
    between and after them (contiguous views, as arena rows are)."""
    GUARD = 1234.5

    def __init__(self, shapes, dtype, device, gap=7):
        sizes = [math.prod(s) for s in shapes]
        self.buf = torch.full((sum(sizes) + gap * (len(shapes) + 1),), self.GUARD, dtype=dtype, device=device)
        self.guard = torch.ones(self.buf.shape, dtype=torch.bool, device=device)
        self.views, off = [], gap
        for s, n in zip(shapes, sizes):
            self.views.append(self.buf[off: off + n].view(s).fill_(float("nan")))
            self.guard[off: off + n] = False
            off += n + gap

    def assert_guards(self, what=""):
        assert (self.buf[self.guard] == self.GUARD).all(), (what, "a write outside the outputs")


# ---- acceptance ------------------------------------------------------------------------------------------------------
# Fractions of the yardstick's error a kernel may make.  The 3xTF32 conv-net kernel measures at most 0.02 of the
# 1xTF32 yardstick (H100, all three cluster instantiations).  The bf16 MLP training kernel measures at most 0.14 of
# the faithful-vs-exact yardstick (per tensor and per block; H100): the SFU sine and exp and the fp32 tensor-core
# accumulation move a small fraction of the bf16 roundings by one ulp.  A zeroed 16 x 8 tile, a missing 16-row
# k-step or a stored-instead-of-added tile measures 9x or more (tests/test_kernel_oracles.py).
#
# The fp32 CUDA-core kernels (``convnet_generic_kernel<float, ...>``, ``mlp_generic_*_kernel<float>``) are held to
# TF32_POINT_FRAC of the error the exact math makes at the TF32 rounding of its inputs (``convnet_tf32_point``, and
# ``mlp_fp64`` at ``round_tf32`` of the parameters, the rows and dL/dout).  fp32 autograd measures at most 0.032
# (conv net) and 0.009 (MLP) of it on CPU; a partial batch scaled by the wrong size, a dropped sample or a dropped
# conv-gradient partition measure 200x or more, a 32-row CTA missing from a weight gradient 4.3x
# (tests/test_kernel_oracles.py).
CONVNET_FRAC = 0.1
MLP_FRAC = 0.3
TF32_POINT_FRAC = 0.1


def _block_errors(d: torch.Tensor, block) -> torch.Tensor:
    """Frobenius norm of every ``block`` (16 x 8 for a matrix, 128 entries for a vector) of ``d``."""
    if d.dim() == 1:
        n = -(-d.numel() // block[0] // block[1]) * block[0] * block[1]
        return F.pad(d, (0, n - d.numel())).reshape(-1, block[0] * block[1]).norm(dim=1)
    d = d.reshape(d.shape[0], -1)
    R, C = -(-d.shape[0] // block[0]) * block[0], -(-d.shape[1] // block[1]) * block[1]
    d = F.pad(d, (0, C - d.shape[1], 0, R - d.shape[0]))
    return d.reshape(R // block[0], block[0], C // block[1], block[1]).pow(2).sum((1, 3)).sqrt().flatten()


def error_ratios(got, ref, yardstick, spec=None, block=(16, 8)):
    """``{name: (norm ratio, block ratio)}``: the kernel's error over the yardstick's, as the norm of the whole tensor
    and as the largest 16 x 8 block.  ``got`` / ``ref`` / ``yardstick`` are flat arena rows (with ``spec``) or dicts
    of tensors."""
    if spec is not None:
        names = [f"p{i}" for i in range(len(spec.param_shapes()))]
        got, ref, yardstick = (dict(zip(names, unflatten(t, spec))) for t in (got, ref, yardstick))
    out = {}
    for k in ref:
        g, r, y = (t[k].to(torch.float64) for t in (got, ref, yardstick))
        e_g, e_y = _block_errors(g - r, block), _block_errors(y - r, block)
        out[k] = (_ratio(e_g.norm(), e_y.norm()), _ratio(e_g.max(), e_y.max()))
    return out


def _ratio(a, b):
    a, b = float(a), float(b)
    return 0.0 if a == 0.0 else (a / b if b > 0.0 else math.inf)


def assert_close_to_oracle(got, ref, yardstick, frac, spec=None, block=(16, 8)):
    """Every tensor's error against ``ref`` is at most ``frac`` times the yardstick's error, as a norm over the whole
    tensor and as the largest 16 x 8 block (a zeroed or doubled tile stands out in its block even where the tensor's
    norm barely moves).  Returns the ratios."""
    rat = error_ratios(got, ref, yardstick, spec, block)
    bad = {k: v for k, v in rat.items() if max(v) > frac}
    assert not bad, f"error / yardstick error above {frac}: {bad}"
    return rat
