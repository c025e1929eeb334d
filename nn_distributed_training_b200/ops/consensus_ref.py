"""PyTorch reference implementation of every consensus op.

These are the numerical oracles for the fused sm_90a kernels in
``csrc/consensus.cu`` and the execution path on CPU / gloo.  Each function works
on arena rows ``[L, n_pad]`` of the local nodes and, where neighbor data is
needed, on the gathered matrix ``[N, n_pad]`` of all nodes' published rows.

Equations: SURVEY Appendix D; reference call sites optimizers/dinno.py:74-125,
optimizers/dsgd.py:34-58, optimizers/dsgt.py:33-103.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np
import torch

ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8
ADAMW_WEIGHT_DECAY = 1e-2  # torch.optim.AdamW default, used by the reference as-is


# ---------------------------------------------------------------- DiNNO ----
def dinno_exchange_(theta_k: torch.Tensor, theta_all: torch.Tensor, adj_rows: torch.Tensor,
                    deg: torch.Tensor, rho: float, dual: torch.Tensor, delta: torch.Tensor):
    """Dual ascent and proximal-centre build for one round.

    ``delta_i = sum_j (theta_j^k - theta_i^k)``; ``dual_i -= rho delta_i``
    (optimizers/dinno.py:123).  ``delta`` is the only neighbor-dependent term the
    primal gradient needs (closed form of ``rho sum_j |theta-(theta_i^k+theta_j^k)/2|^2``,
    optimizers/dinno.py:85-89,124), so no ``[d_i, n]`` stack is ever built.
    Differences are accumulated per neighbor (not ``sum_j theta_j - d_i theta_i``),
    as the fused kernel and the reference do, so the terms vanish exactly at
    consensus and keep their precision near it.  ``deg`` is implied by
    ``adj_rows`` and kept for the call signature.
    """
    a = adj_rows.to(theta_all.dtype)
    delta.zero_()
    for j in torch.nonzero(a.any(0)).flatten().tolist():
        delta.add_(torch.where(a[:, j: j + 1] != 0, theta_all[j] - theta_k, 0.0))
    dual.add_(delta, alpha=-rho)


def dinno_grad(theta: torch.Tensor, theta_k: torch.Tensor, grad: torch.Tensor, dual: torch.Tensor,
               delta: torch.Tensor, deg: torch.Tensor, rho: float) -> torch.Tensor:
    """Gradient of ``loss + theta.dual + rho sum_j |theta - (theta_i^k+theta_j^k)/2|^2``
    = ``grad + dual + 2 rho d_i (theta - theta_i^k) - rho delta_i``."""
    d = deg.to(theta.dtype).unsqueeze(1)
    return grad + dual + (2.0 * rho) * d * (theta - theta_k) - rho * delta


def optimizer_step_(theta: torch.Tensor, g: torch.Tensor, kind: str, lr: float,
                    m: Optional[torch.Tensor], v: Optional[torch.Tensor], t: int):
    """One torch.optim-equivalent step (Adam / AdamW / SGD defaults), ``t`` is the
    1-based step count used for bias correction."""
    if kind == "sgd":
        theta.add_(g, alpha=-lr)
        return
    if kind == "adamw":
        theta.mul_(1.0 - lr * ADAMW_WEIGHT_DECAY)
    elif kind != "adam":
        raise NameError("DiNNO primal optimizer is unknown.")
    m.mul_(ADAM_BETA1).add_(g, alpha=1.0 - ADAM_BETA1)
    v.mul_(ADAM_BETA2).addcmul_(g, g, value=1.0 - ADAM_BETA2)
    bc1 = 1.0 - ADAM_BETA1 ** t
    bc2 = 1.0 - ADAM_BETA2 ** t
    denom = (v.sqrt() / math.sqrt(bc2)).add_(ADAM_EPS)
    theta.addcdiv_(m, denom, value=-(lr / bc1))


# ----------------------------------------------------------------- DSGD ----
def dsgd_mix(theta_all: torch.Tensor, w_rows: torch.Tensor) -> torch.Tensor:
    """Jacobi mixing ``theta_i <- sum_j W_ij theta_j`` for the local rows."""
    return w_rows.to(theta_all.dtype) @ theta_all


def dsgd_step_(theta: torch.Tensor, grad: torch.Tensor, alpha: float):
    theta.add_(grad, alpha=-alpha)


def dsgd_alpha(alpha_prev: float, mu: float) -> float:
    """``alpha_k = alpha_{k-1} (1 - mu alpha_{k-1})`` (optimizers/dsgd.py:34)."""
    return alpha_prev * (1.0 - mu * alpha_prev)


# ----------------------------------------------------------------- DSGT ----
def dsgt_mix(theta_all: torch.Tensor, y_all: torch.Tensor, w_rows: torch.Tensor, alpha: float) -> torch.Tensor:
    """``theta_i <- sum_j W_ij (theta_j - alpha y_j)``."""
    return w_rows.to(theta_all.dtype) @ (theta_all - alpha * y_all)


def dsgt_track(y_all: torch.Tensor, w_rows: torch.Tensor, g_new: torch.Tensor, g_old: torch.Tensor) -> torch.Tensor:
    """``y_i <- sum_j W_ij y_j + g_i^{new} - g_i^{old}``."""
    return w_rows.to(y_all.dtype) @ y_all + g_new - g_old


# ------------------------------------------------------ Exact Diffusion ----
def ed_weights(W):
    """``A = (I + W) / 2`` of a float64 Metropolis matrix: the combine weights of Exact Diffusion."""
    return 0.5 * (np.eye(W.shape[0]) + W)


def ed_step_(theta: torch.Tensor, psi: torch.Tensor, grad: torch.Tensor, alpha: float):
    """``psi' = theta - alpha g``; ``theta <- psi' + (theta - psi)``; ``psi <- psi'``, on the mixed rows ``theta``."""
    corr = theta - psi
    psi.copy_(theta).add_(grad, alpha=-alpha)
    theta.copy_(psi).add_(corr)


# ------------------------------------------------------------- metrics ----
def consensus_error(theta_all: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Pairwise and to-mean distances of L2-normalised parameter rows
    (problems/dist_mnist_problem.py:155-169)."""
    th = torch.nn.functional.normalize(theta_all, dim=1)
    d_all = torch.cdist(th, th)
    d_mean = torch.cdist(th, th.mean(dim=0, keepdim=True))
    return d_all, d_mean


# ----------------------------------------- reference-order (Gauss-Seidel) ----
def dsgd_mix_sequential_(theta: torch.Tensor, W: torch.Tensor, neighbors):
    """In-place sweep in node index order exactly as optimizers/dsgd.py:37-46:
    node i sees already-mixed rows of neighbors j < i.  Single-process only."""
    for i, nbrs in enumerate(neighbors):
        theta[i].mul_(W[i, i])
        for j in nbrs:
            theta[i].add_(W[i, j] * theta[j])


def dsgt_mix_sequential_(theta: torch.Tensor, y: torch.Tensor, W: torch.Tensor, neighbors, alpha: float):
    """optimizers/dsgt.py:58-75: sequential in theta, round-k y everywhere."""
    for i, nbrs in enumerate(neighbors):
        theta[i].mul_(W[i, i])
        theta[i].add_(y[i], alpha=-alpha * float(W[i, i]))
        for j in nbrs:
            theta[i].add_(theta[j], alpha=float(W[i, j]))
            theta[i].add_(y[j], alpha=-alpha * float(W[i, j]))


def dsgt_track_sequential_row_(i: int, y: torch.Tensor, W: torch.Tensor, nbrs, g_new: torch.Tensor, g_old: torch.Tensor):
    """optimizers/dsgt.py:87-98 for one node (sequential in y)."""
    y[i].mul_(W[i, i])
    for j in nbrs:
        y[i].add_(y[j], alpha=float(W[i, j]))
    y[i].add_(g_new)
    y[i].add_(g_old, alpha=-1.0)
