"""Plain feed-forward nets (reference: models/relu_nn.py:4-116, and the RL copy
RL/dist_rl/model.py:6-45 which additionally coerces numpy observations)."""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from .spec import MLPSpec


def _stack(shape, act_factory, act_on_last, dtype):
    kw = {} if dtype is None else {"dtype": dtype}
    mods = []
    last = len(shape) - 2
    for li in range(len(shape) - 1):
        mods.append(nn.Linear(shape[li], shape[li + 1], **kw))
        if li != last or act_on_last:
            mods.append(act_factory())
    return nn.Sequential(*mods)


class _FFNet(nn.Module):
    _act = "relu"
    _act_on_last = False

    def __init__(self, shape, dtype=None, coerce_numpy=False):
        super().__init__()
        self.shape = [int(s) for s in shape]
        self.coerce_numpy = coerce_numpy
        a = self._act
        self.spec = MLPSpec(tuple(self.shape), first=a, hidden=a,
                            last=a if self._act_on_last else "none")
        factory = {"relu": lambda: nn.ReLU(inplace=True), "tanh": nn.Tanh, "sigmoid": nn.Sigmoid}[a]
        self.seq = _stack(self.shape, factory, self._act_on_last, dtype)

    def _layer_acts(self):
        n = len(self.shape) - 1
        return [self._act if (li != n - 1 or self._act_on_last) else "none" for li in range(n)]

    def forward(self, x):
        if self.coerce_numpy and isinstance(x, np.ndarray):
            p = next(self.parameters())
            x = torch.as_tensor(x, dtype=p.dtype, device=p.device)
        if x.is_cuda:
            # CUDA: the whole network is one fused forward launch and one fused backward launch
            # (ops/csrc/mlp_generic.cu); NNDT_FUSED_MLP=0 or an unsupported width falls back to nn.Sequential loudly
            from ..ops import mlp_generic as mg
            acts = self._layer_acts()
            if mg.enabled() and mg.supported(self.shape, acts, x.dtype):
                params = list(self.seq.parameters())
                if not mg.arguments_match(x, params, self.shape):
                    return self.seq(x)          # a dtype, device or width mismatch: nn.Sequential's own error
                return mg.fused_mlp(x, params, self.shape, acts)
            if not getattr(self, "_warned", False):
                self._warned = True
                print(f"[nndt] WARNING: {type(self).__name__}{self.shape} ({x.dtype}) runs nn.Sequential (cuBLAS) on CUDA: "
                      "no fused kernel for this shape / dtype or NNDT_FUSED_MLP=0", flush=True)
        return self.seq(x)


class FFReLUNet(_FFNet):
    """(Linear+ReLU)*(L-1) -> Linear (no activation on the output layer)."""
    _act, _act_on_last = "relu", False


class FFTanhNet(_FFNet):
    """Tanh after every layer including the last (reference :62-64)."""
    _act, _act_on_last = "tanh", True


class FFSigmoidNet(_FFNet):
    """Sigmoid after every layer including the last (reference :100-102)."""
    _act, _act_on_last = "sigmoid", True
