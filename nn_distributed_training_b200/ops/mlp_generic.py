"""Module-level fused forward / backward of plain feed-forward nets (csrc/mlp_generic.cu).

``fused_mlp(x, params, shape, acts)`` is a ``torch.autograd.Function``: ONE forward launch for the whole network (every
layer's activation saved for the backward pass) and ONE backward launch producing every parameter gradient, instead of
the 2-3 ATen launches per layer and direction of ``nn.Sequential`` (reference models: models/relu_nn.py:4-116,
RL/dist_rl/model.py:6-45).  ``params`` is the ordinary list of ``nn.Linear`` weights and biases; they are packed into one
flat vector with ``torch.cat`` (differentiable), so free-standing modules and arena-attached ones work the same way.
"""
from __future__ import annotations

import os
from typing import List, Sequence

import torch

from . import load_ext

ACT = {"none": 0, "relu": 1, "tanh": 2, "sigmoid": 3}
MAX_WIDTH, MAX_LAYERS = 256, 8


def supported(shape: Sequence[int], acts: Sequence[str], dtype) -> bool:
    return (2 <= len(shape) <= MAX_LAYERS + 1 and all(1 <= int(s) <= MAX_WIDTH for s in shape)
            and all(a in ACT for a in acts) and dtype in (torch.float32, torch.float64))


def arguments_match(x: torch.Tensor, params: Sequence[torch.Tensor], shape: Sequence[int]) -> bool:
    """The kernels read ``x`` and the parameters as raw ``x.dtype`` arrays on ``x``'s device, ``shape[0]`` values per
    row: a parameter of another dtype or device, or a row of another width, would be read as garbage or out of bounds.
    Callers run ``nn.Sequential`` instead, which raises its own error for the mismatch."""
    return (x.shape[-1] == int(shape[0])
            and all(p.dtype == x.dtype and p.device == x.device for p in params))


def enabled() -> bool:
    return os.environ.get("NNDT_FUSED_MLP", "1") != "0"


def _desc(shape, acts, dtype):
    w_off, b_off, off = [], [], 0
    for l in range(len(shape) - 1):
        w_off.append(off); off += shape[l + 1] * shape[l]
        b_off.append(off); off += shape[l + 1]
    return dict(dims=[int(s) for s in shape], act=[ACT[a] for a in acts], w_off=w_off, b_off=b_off,
                dtype64=int(dtype == torch.float64)), off


class _FusedMLP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, flat, shape, acts):
        ext = load_ext(required=True)
        x = x.contiguous()
        flat = flat.contiguous()
        M = x.shape[0]
        d, n = _desc(shape, acts, x.dtype)
        assert flat.numel() == n
        buf = torch.empty(M, sum(shape[1:]), dtype=x.dtype, device=x.device)
        d.update(x=x.data_ptr(), params=flat.data_ptr(), M=M, acts=buf.data_ptr())
        ext.mlp_generic_forward(d)
        ctx.save_for_backward(x, flat, buf)
        ctx.desc = (tuple(shape), tuple(acts))
        return buf[:, buf.shape[1] - shape[-1]:]

    @staticmethod
    def backward(ctx, gout):
        ext = load_ext(required=True)
        x, flat, buf = ctx.saved_tensors
        shape, acts = ctx.desc
        d, _ = _desc(shape, acts, x.dtype)
        gout = gout.contiguous()
        gflat = torch.zeros_like(flat)
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        d.update(x=x.data_ptr(), params=flat.data_ptr(), M=x.shape[0], acts=buf.data_ptr(), gout=gout.data_ptr(),
                 gparams=gflat.data_ptr(), gx=None if gx is None else gx.data_ptr())
        ext.mlp_generic_backward(d)
        return gx, gflat, None, None


def fused_mlp(x: torch.Tensor, params: List[torch.Tensor], shape: Sequence[int], acts: Sequence[str]) -> torch.Tensor:
    """``x [..., d0]`` -> ``[..., d_last]``; ``params = [W0, b0, W1, b1, ...]`` (``nn.Linear`` layout)."""
    lead = x.shape[:-1]
    x2 = x.reshape(-1, x.shape[-1])
    if x2.shape[0] == 0:
        return x.new_zeros(*lead, shape[-1])
    flat = torch.cat([p.reshape(-1) for p in params])
    out = _FusedMLP.apply(x2, flat, tuple(int(s) for s in shape), tuple(acts))
    return out.reshape(*lead, shape[-1])
