"""Which density networks, losses and dtypes the fused MLP kernels accept (CPU: no kernel is launched)."""
import itertools

import pytest
import torch

from nn_distributed_training_b200.models.spec import MLPSpec
from nn_distributed_training_b200.ops import mlp_kernel_supports
from nn_distributed_training_b200.ops.mlp_fused import supports

SHAPES = [([2, 64, 64, 64, 64, 1], True), ([2, 128, 64, 64, 64, 1], True), ([2, 256, 64, 64, 64, 1], True),
          ([2, 96, 64, 64, 64, 1], False), ([2, 256, 64, 64, 1], False), ([3, 256, 64, 64, 64, 1], False),
          ([2, 256, 64, 64, 64, 2], False), ([2, 256, 128, 64, 64, 1], False)]
NETS = [("sin_relu", "sigmoid"), ("relu", "none")]
LOSSES = [(torch.nn.BCELoss(), True), (torch.nn.MSELoss(), True), (torch.nn.L1Loss(), True),
          (torch.nn.MSELoss(reduction="sum"), False), (torch.nn.NLLLoss(), False)]
DTYPES = [(torch.float32, True), (torch.float64, True), (torch.float16, False), (torch.bfloat16, False)]


@pytest.mark.parametrize("shape,shape_ok", SHAPES)
def test_supports_dtype_shape_loss(shape, shape_ok):
    for (first, last), (loss, loss_ok), (dtype, dtype_ok) in itertools.product(NETS, LOSSES, DTYPES):
        spec = MLPSpec(shape, first=first, hidden="relu", last=last, scale=0.05)
        want = shape_ok and loss_ok and dtype_ok
        assert supports(spec, loss, dtype) == want, (shape, first, type(loss).__name__, dtype)
        assert mlp_kernel_supports(spec, loss, dtype) == want


def test_supports_defaults_to_float32():
    spec = MLPSpec([2, 256, 64, 64, 64, 1], first="sin_relu", hidden="relu", last="sigmoid", scale=0.05)
    assert supports(spec, torch.nn.BCELoss()) and mlp_kernel_supports(spec, torch.nn.BCELoss())


def test_supports_rejects_other_hidden_activations():
    spec = MLPSpec([2, 256, 64, 64, 64, 1], first="sin_relu", hidden="tanh", last="sigmoid", scale=0.05)
    for dtype in (torch.float32, torch.float64):
        assert not supports(spec, torch.nn.BCELoss(), dtype)
