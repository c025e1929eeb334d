"""Generalized advantage estimation, GAE(lambda) (Schulman et al. 2016), for the PPO trainers' torch update path.

The batch rows are ``r = (blk * T + c) * E + e``: blocks of ``T`` cycles of ``E`` worlds, each block one episode that
ends in a terminal step (the rollouts do not bootstrap a truncated episode).  Per (block, world):

    delta_c = r_c + gamma * V_{c+1} - V_c,    A_c = delta_c + gamma * lam * A_{c+1},    V_T = A_T = 0,

and ``G = A + V`` is the critic's target (the lambda-return).  ``lam = 1`` gives ``A = rtgs - V``, ``lam = 0`` the
one-step TD residual.  Every product and sum is its own elementwise op in the order written, which is the operation
order of the sm_90a scan (ops/csrc/ppo_update.cu: gae_kernel), so both paths give the same bits from the same ``V``.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch


def check_gae_lambda(value) -> Optional[float]:
    """``None`` (Monte-Carlo advantages ``rtgs - V``) or a finite number in [0, 1], as a float; anything else,
    a bool included, raises ``ValueError``."""
    if value is None:
        return None
    if isinstance(value, bool) or not isinstance(value, (int, float)) or not math.isfinite(value) \
            or not 0.0 <= value <= 1.0:
        raise ValueError(f"gae_lambda must be None or a finite float in [0, 1], not {value!r}")
    return float(value)


def gae(rews: torch.Tensor, values: torch.Tensor, gamma: float, lam: float, T: int,
        E: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(A, G)`` of GAE(lambda) for rewards and values ``[..., R]`` in the row order above (``T * E`` dividing R)."""
    shape = rews.shape
    if shape[-1] % (T * E):
        raise ValueError(f"T * E = {T} * {E} must divide R = {shape[-1]}")
    r = rews.reshape(-1, T, E)
    v = values.reshape(-1, T, E)
    A = torch.empty_like(r)
    a = torch.zeros_like(r[:, 0])
    vn = torch.zeros_like(r[:, 0])
    gl = gamma * lam
    for c in range(T - 1, -1, -1):
        delta = (r[:, c] + gamma * vn) - v[:, c]
        a = delta + gl * a
        A[:, c] = a
        vn = v[:, c]
    return A.reshape(shape), (A + v).reshape(shape)
