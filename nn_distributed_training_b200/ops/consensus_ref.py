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
from typing import List, Optional, Tuple

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


# ----------------------------------------------------------- Gossip-PGA ----
def pga_mean_(theta: torch.Tensor, theta_all: torch.Tensor) -> None:
    """The global round's mix of Gossip-PGA: every local row of ``theta`` becomes the mean of all N rows of
    ``theta_all``, accumulated in float64 in node order and cast once to the arena dtype (the fused ``pga_mix`` on one
    GPU computes the same bits)."""
    s = torch.zeros(theta_all.shape[1], dtype=torch.float64, device=theta_all.device)
    for j in range(theta_all.shape[0]):
        s += theta_all[j].double()
    theta.copy_((s / theta_all.shape[0]).to(theta.dtype).expand_as(theta))


# ---------------------------------------------------------------- SlowMo ----
def slowmo_outer_(theta: torch.Tensor, anchor: torch.Tensor, u: torch.Tensor, m: Optional[torch.Tensor], gamma: float,
                  slow_lr: float, slow_momentum: float) -> None:
    """SlowMo's outer update on a global round, with ``theta`` holding the mean ``xbar`` (``pga_mean_``):
    ``u <- slow_momentum u + (anchor - xbar) / gamma``, ``anchor <- anchor - (slow_lr gamma) u``, ``theta <- anchor``
    and ``m <- 0`` (when given).  Evaluated in float64 from the stored rows, every operation rounded on its own, and
    each stored row rounded once; ``gamma`` is taken in the arena dtype first, as the fused kernel reads it from the
    schedule (csrc/consensus.cu: slowmo_outer_kernel computes the same bits)."""
    gamma = float(torch.tensor(gamma, dtype=theta.dtype))
    a = anchor.double()
    un = u.double() * slow_momentum + (a - theta.double()) / gamma
    u.copy_(un)
    anchor.copy_(a - (slow_lr * gamma) * un)
    theta.copy_(anchor)
    if m is not None:
        m.zero_()


# ---------------------------------------------------------------- DeTAG ----
def mixing_lambda(W: np.ndarray) -> float:
    """``max |eig(W - 11^T / N)|`` of a symmetric mixing matrix, in float64 (0 for one node and the complete graph)."""
    N = W.shape[0]
    if N == 1:
        return 0.0
    return float(np.abs(np.linalg.eigvalsh(np.asarray(W, dtype=np.float64) - 1.0 / N)).max())


def chebyshev_weights(lam: float, K: int, accelerate: bool = True) -> List[float]:
    """The sub-step weights ``w_0 .. w_{K-1}`` of Chebyshev-accelerated gossip, in float64: ``w_0 = 1``,
    ``w_1 = 2 / (2 - lam^2)``, ``w_s = 1 / (1 - lam^2 w_{s-1} / 4)``.  Every ``w_s = 1`` without acceleration (plain K-step
    gossip) and when ``lam = 0``."""
    out = [1.0] * K
    if accelerate and lam > 0.0:
        l2 = lam * lam
        for s in range(1, K):
            out[s] = 2.0 / (2.0 - l2) if s == 1 else 1.0 / (1.0 - l2 * out[s - 1] / 4.0)
    return out


def ag_gossip(x_all: torch.Tensor, x_prev: Optional[torch.Tensor], w_rows: torch.Tensor, omega: float) -> torch.Tensor:
    """One gossip sub-step of the local rows: ``M = sum_j W_ij X_j`` and ``X_prev + omega (M - X_prev)`` (``omega == 1``:
    ``M``, and ``x_prev`` is not read)."""
    m = dsgd_mix(x_all, w_rows)
    if omega == 1.0:
        return m
    return x_prev + omega * (m - x_prev)


def detag_track_(y: torch.Tensor, g_old: torch.Tensor, ymix: torch.Tensor, grad: torch.Tensor, theta: torch.Tensor,
                 alpha: float) -> torch.Tensor:
    """``y <- Y_K + (g - g_old)``, ``g_old <- g``; returns the row to publish, ``z = theta - alpha y``."""
    y.copy_(ymix + (grad - g_old))
    g_old.copy_(grad)
    return theta - alpha * y


# -------------------------------------------------------------- GT-HSGD ----
def hsgd_track_(y: torch.Tensor, v: torch.Tensor, theta_prev: torch.Tensor, y_all: torch.Tensor, w_rows: torch.Tensor,
                grad: torch.Tensor, grad_prev: torch.Tensor, theta: torch.Tensor, omb: float, first: bool) -> None:
    """The tracking step of GT-HSGD on the local rows: ``v' = g`` (``first``, round 0) or ``g + omb (v - gp)`` with
    ``omb = 1 - beta``, then ``y <- sum_j W_ij y_j + v' - v`` (``dsgt_track`` with v in place of the gradient),
    ``v <- v'`` and ``theta_prev <- theta``."""
    vn = grad.clone() if first else grad + omb * (v - grad_prev)
    y.copy_(dsgt_track(y_all, w_rows, vn, v))
    v.copy_(vn)
    theta_prev.copy_(theta)


# ------------------------------------------------------- cross-gradient ----
def xg_coefs(W: np.ndarray, neighbors, lam: float, lo: int, L: int, dmax: int) -> Tuple[np.ndarray, np.ndarray]:
    """float64 weights of the aggregated direction of local nodes ``lo .. lo + L - 1``: ``coef0[l] = (1 - lam) + lam
    W_ii`` and ``coef[l, e] = lam W_{i j_e}`` in table order (``neighbors[i]``), 0 past deg_i."""
    coef0 = np.zeros(L)
    coef = np.zeros((L, dmax))
    for l in range(L):
        i = lo + l
        coef0[l] = (1.0 - lam) + lam * W[i, i]
        for e, j in enumerate(neighbors[i]):
            coef[l, e] = lam * W[i, j]
    return coef0, coef


def xg_cross_points(theta_all: torch.Tensor, src_node: torch.Tensor, live: torch.Tensor, lo: int) -> torch.Tensor:
    """``[dmax, L, n_pad]``: slot e of local node l is neighbor j_e's row (``src_node[l, e]``) of ``theta_all``, or the
    node's own row past deg_l (``live`` false)."""
    L, dmax = src_node.shape
    own = theta_all[lo: lo + L]
    return torch.stack([torch.where(live[:, e, None], theta_all[src_node[:, e]], own) for e in range(dmax)])


def xg_received(grad_x_all: torch.Tensor, src_node: torch.Tensor, src_slot: torch.Tensor,
                live: torch.Tensor) -> torch.Tensor:
    """``[L, dmax, n_pad]``: ``g_{j_e -> i}``, the gradient neighbor j_e took at this node's row, picked from every
    node's cross gradients ``grad_x_all`` (``[dmax, N, n_pad]``) at ``[src_slot, src_node]`` (its reverse slot); zero
    past deg_i."""
    r = grad_x_all[src_slot, src_node]
    return torch.where(live[:, :, None], r, torch.zeros((), dtype=r.dtype))


def xg_step_(theta: torch.Tensor, xmix: torch.Tensor, grad: torch.Tensor, recv: torch.Tensor, coef0: torch.Tensor,
             coef: torch.Tensor, alpha: float) -> torch.Tensor:
    """``d = coef0 g + sum_e coef_e g_{j_e -> i}`` in float64 (own term first, then table order), rounded once to the
    arena dtype; then ``theta = xmix - alpha d`` (dsgd_step_).  ``coef0`` ``[L]`` and ``coef`` ``[L, dmax]`` are
    float64; ``recv`` ``[L, dmax, n_pad]``.  Returns d."""
    d = coef0[:, None] * grad.double()
    for e in range(recv.shape[1]):
        d = d + coef[:, e, None] * recv[:, e].double()
    d = d.to(theta.dtype)
    theta.copy_(xmix)
    dsgd_step_(theta, d, alpha)
    return d


# ------------------------------------------------------ Exact Diffusion ----
def ed_weights(W):
    """``A = (I + W) / 2`` of a float64 Metropolis matrix: the combine weights of Exact Diffusion."""
    return 0.5 * (np.eye(W.shape[0]) + W)


def ed_step_(theta: torch.Tensor, psi: torch.Tensor, grad: torch.Tensor, alpha: float):
    """``psi' = theta - alpha g``; ``theta <- psi' + (theta - psi)``; ``psi <- psi'``, on the mixed rows ``theta``."""
    corr = theta - psi
    psi.copy_(theta).add_(grad, alpha=-alpha)
    theta.copy_(psi).add_(corr)


# --------------------------------------------------- DSGD with momentum ----
def dsgdm_step_(theta: torch.Tensor, m: torch.Tensor, x_prev: Optional[torch.Tensor], grad: torch.Tensor, alpha: float,
                alpha_prev: float, beta: float, quasi_global: bool, nesterov: bool, first: bool):
    """The momentum step on the mixed rows ``x = theta`` (``first``: round 0, where ``m`` and ``x_prev`` are not read).

    local:         ``m <- beta m + g``
    quasi-global:  ``m <- beta m + (1 - beta) (x_prev - x) / alpha_prev`` after round 0 (``m`` holds mhat, 0 in round
                   0); the step's momentum is ``beta mhat + g``; ``x_prev <- x``
    both:          ``theta <- x - alpha (nesterov ? g + beta mom : mom)``"""
    if quasi_global:
        if first:
            m.zero_()
        else:
            m.mul_(beta).add_((x_prev - theta) / alpha_prev, alpha=1.0 - beta)
        x_prev.copy_(theta)
        mom = grad.add(m, alpha=beta)
    else:
        if first:
            m.copy_(grad)
        else:
            m.mul_(beta).add_(grad)
        mom = m
    theta.add_(grad.add(mom, alpha=beta) if nesterov else mom, alpha=-alpha)


# ------------------------------------------------------------ CHOCO-SGD ----
# Code rows (the byte layout of csrc/consensus.h, the only other place it is written).  A row of n_pad elements is cut
# into nb = n_pad / 32 blocks of 32; scales are in the arena dtype T:
#   none: [n_pad] T                        v itself
#   int8: [n_pad] int8, [nb] T scales      scale = max|v| / 127, code = clamp(rint(v / scale), -127, 127), dec = code scale
#   sign: [nb] uint32 words, [nb] T        bit e % 32 of word e // 32 set when v_e >= 0; scale = sum|v| / n_live over the
#                                          live elements, dec = +-scale on live elements and 0 on padding and holes
#   topk: [k] T values, [k] uint32 indices the k live elements of largest |v| (choco_topk_select), indices ascending,
#         zero padding to a multiple of 16 B  values exact (not rescaled); dec = v at the indices, 0 elsewhere
# The arithmetic is the kernel's: divisions and the decode product are single IEEE operations, round half to even, and
# the sign scale's sum runs in the kernel's order (elements of a lane in turn, then halving over the 32 / VEC lanes
# of the block), so both paths produce the same bytes from the same v.
CHOCO_COMPRESSORS = ("none", "int8", "sign", "topk")
CHOCO_CODE = {"none": 0, "int8": 1, "sign": 2, "topk": 3}
CHOCO_BLOCK = 32
CHOCO_VEC = {torch.float32: 4, torch.float64: 2}      # elements per thread in the kernels (16-byte vectors)
TOPK_RATIO_DEFAULT = 0.01


def choco_topk_k(ratio: float, n_live: int) -> int:
    """Entries a top-k code row keeps: ``max(1, ceil(ratio * n_live))`` of the ``n_live`` parameter elements."""
    if not 0.0 < float(ratio) <= 1.0:
        raise ValueError(f"topk_ratio must be in (0, 1] (got {ratio!r})")
    return max(1, math.ceil(float(ratio) * int(n_live)))


def choco_k(conf, compressor: str, live: torch.Tensor, alg: str) -> Optional[int]:
    """The k of a ``topk`` compressor from an optimizer config (``topk_ratio``, default ``TOPK_RATIO_DEFAULT``), None
    for the other compressors; ``topk_ratio`` with another compressor is refused."""
    ratio = conf.get("topk_ratio")
    if compressor != "topk":
        if ratio is not None:
            raise ValueError(f"{alg} topk_ratio applies to compressor topk only (compressor is {compressor!r})")
        return None
    return choco_topk_k(TOPK_RATIO_DEFAULT if ratio is None else ratio, int(live.sum()))


def choco_code_bytes(compressor: str, n_pad: int, dtype: torch.dtype, k: Optional[int] = None) -> int:
    """Bytes of one code row (``k``: entries of a top-k row)."""
    s = torch.empty((), dtype=dtype).element_size()
    nb = n_pad // CHOCO_BLOCK
    if compressor == "topk":
        return -(-k * (s + 4) // 16) * 16
    return {"none": n_pad * s, "int8": n_pad + nb * s, "sign": 4 * nb + nb * s}[compressor]


def choco_topk_keys(v: torch.Tensor, live: torch.Tensor) -> torch.Tensor:
    """Selection keys of ``v [L, n_pad]``: the IEEE bit pattern with the sign bit cleared (so ``+0`` and ``-0`` tie and
    the order is exact in both dtypes) as int64, ``-1`` on padding and holes (never selected)."""
    if v.dtype == torch.float64:
        key = v.contiguous().view(torch.int64) & 0x7FFFFFFFFFFFFFFF
    else:
        key = (v.contiguous().view(torch.int32) & 0x7FFFFFFF).to(torch.int64)
    return torch.where(live.to(v.device), key, torch.full_like(key, -1))


def choco_topk_select(v: torch.Tensor, live: torch.Tensor, k: int) -> torch.Tensor:
    """``[L, k]`` indices (int64, ascending) of the k live elements of each row with the largest ``|v|``; ties go to the
    smaller index."""
    order = torch.sort(choco_topk_keys(v, live), dim=1, descending=True, stable=True).indices
    return order[:, :k].sort(dim=1).values


def choco_live(layout) -> torch.Tensor:
    """``[n_pad]`` bool: True on parameter elements, False on row padding and slot-alignment holes."""
    live = torch.zeros(layout.n_pad, dtype=torch.bool)
    for s in layout.slots:
        live[s.offset: s.offset + s.numel] = True
    return live


def choco_live_words(live: torch.Tensor) -> torch.Tensor:
    """The ``[n_pad / 32]`` bit mask the kernels read (bit e % 32 of word e // 32), as int32."""
    bits = np.packbits(live.cpu().numpy().astype(np.uint8), bitorder="little")
    return torch.from_numpy(bits.view(np.int32).copy())


def _blocks(x: torch.Tensor) -> torch.Tensor:
    return x.reshape(x.shape[:-1] + (x.shape[-1] // CHOCO_BLOCK, CHOCO_BLOCK))


def choco_encode(v: torch.Tensor, compressor: str, live: torch.Tensor,
                 k: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Code rows ``[L, code_bytes]`` (uint8) of ``v [L, n_pad]`` and their decoded values ``[L, n_pad]``."""
    L, n_pad = v.shape
    dt = v.dtype
    if compressor == "none":
        return v.contiguous().view(torch.uint8).clone(), v.clone()
    if compressor == "topk":
        idx = choco_topk_select(v, live, k)
        vals = v.gather(1, idx)
        codes = torch.zeros(L, choco_code_bytes("topk", n_pad, dt, k), dtype=torch.uint8, device=v.device)
        s = v.element_size()
        codes[:, : k * s] = vals.contiguous().view(torch.uint8)
        codes[:, k * s: k * (s + 4)] = idx.to(torch.int32).contiguous().view(torch.uint8)
        return codes, torch.zeros_like(v).scatter_(1, idx, vals)
    vb = _blocks(v)
    lb = _blocks(live.to(v.device))
    if compressor == "int8":
        m = vb.abs().amax(-1, keepdim=True)
        sc = m / torch.full_like(m, 127.0)           # a tensor divisor: true division, not a reciprocal product
        pos = sc > 0
        q = torch.where(pos, torch.round(vb / torch.where(pos, sc, torch.ones_like(sc))), torch.zeros_like(vb))
        q = q.clamp_(-127.0, 127.0)
        dec = (q * sc).reshape(L, n_pad)
        codes = torch.cat([q.to(torch.int8).reshape(L, n_pad).view(torch.uint8),
                           sc.reshape(L, -1).contiguous().view(torch.uint8)], dim=1)
        return codes, dec
    if compressor != "sign":
        raise ValueError(f"unknown compressor {compressor!r}")
    vec = CHOCO_VEC[dt]
    a = torch.where(lb, vb.abs(), torch.zeros_like(vb)).reshape(L, -1, CHOCO_BLOCK // vec, vec)
    p = a[..., 0]
    for u in range(1, vec):
        p = p + a[..., u]
    while p.shape[-1] > 1:
        h = p.shape[-1] // 2
        p = p[..., :h] + p[..., h:]
    p = p[..., 0]
    nl = lb.sum(-1).to(dt).expand_as(p)
    sc = torch.where(nl > 0, p / torch.where(nl > 0, nl, torch.ones_like(nl)), torch.zeros_like(p))
    bits = vb >= 0
    shifts = torch.arange(CHOCO_BLOCK, device=v.device, dtype=torch.int64)
    words = (bits.to(torch.int64) << shifts).sum(-1)
    wbytes = torch.stack([(words >> (8 * k)) & 255 for k in range(4)], dim=-1).to(torch.uint8).reshape(L, -1)
    scb = sc.unsqueeze(-1)
    dec = torch.where(lb, torch.where(bits, scb, -scb), torch.zeros_like(vb)).reshape(L, n_pad)
    codes = torch.cat([wbytes, sc.contiguous().view(torch.uint8)], dim=1)
    return codes, dec


def choco_decode(codes: torch.Tensor, compressor: str, n_pad: int, dtype: torch.dtype,
                 live: torch.Tensor, k: Optional[int] = None) -> torch.Tensor:
    """``dec(q)`` of code rows ``[R, code_bytes]`` (uint8) -> ``[R, n_pad]`` in ``dtype``."""
    codes = codes.contiguous()
    R = codes.shape[0]
    if compressor == "none":
        return codes.view(dtype).clone()
    if compressor == "topk":
        s = torch.empty((), dtype=dtype).element_size()
        vals = codes[:, : k * s].contiguous().view(dtype)
        idx = codes[:, k * s: k * (s + 4)].contiguous().view(torch.int32).to(torch.int64)
        return torch.zeros(R, n_pad, dtype=dtype, device=codes.device).scatter_(1, idx, vals)
    nb = n_pad // CHOCO_BLOCK
    if compressor == "int8":
        q = codes[:, :n_pad].contiguous().view(torch.int8).to(dtype).reshape(R, nb, CHOCO_BLOCK)
        sc = codes[:, n_pad:].contiguous().view(dtype)
        return (q * sc.unsqueeze(-1)).reshape(R, n_pad)
    if compressor != "sign":
        raise ValueError(f"unknown compressor {compressor!r}")
    wb = codes[:, :4 * nb].to(torch.int64).reshape(R, nb, 4)
    words = wb[..., 0] | (wb[..., 1] << 8) | (wb[..., 2] << 16) | (wb[..., 3] << 24)
    shifts = torch.arange(CHOCO_BLOCK, device=codes.device, dtype=torch.int64)
    bits = ((words.unsqueeze(-1) >> shifts) & 1).bool()
    sc = codes[:, 4 * nb:].contiguous().view(dtype).unsqueeze(-1)
    lb = _blocks(live.to(codes.device))
    zero = torch.zeros((), dtype=dtype, device=codes.device)
    return torch.where(lb, torch.where(bits, sc, -sc), zero).reshape(R, n_pad)


def choco_mix_(theta: torch.Tensor, x_hat: torch.Tensor, s: torch.Tensor, dec_all: torch.Tensor,
               w_rows: torch.Tensor, gamma: float):
    """``s_i += sum_j W_ij dec(q_j)`` (own term included); ``theta_i += gamma (s_i - x_hat_i)``."""
    s.add_(w_rows.to(dec_all.dtype) @ dec_all)
    theta.add_(s - x_hat, alpha=gamma)


def choco_step_(theta: torch.Tensor, x_hat: torch.Tensor, grad: torch.Tensor, alpha: float, compressor: str,
                live: torch.Tensor, k: Optional[int] = None) -> torch.Tensor:
    """``theta -= alpha g``; ``q = Q(theta - x_hat)``; ``x_hat += dec(q)``; returns the code rows ``q`` to publish."""
    theta.add_(grad, alpha=-alpha)
    codes, dec = choco_encode(theta - x_hat, compressor, live, k)
    x_hat.add_(dec)
    return codes


# ------------------------------------------------------------ SPARQ-SGD ----
# A SPARQ row is a CHOCO code row (choco_encode's bytes) followed by a 16-byte tail: uint32 trig, uint32 0, float64 e
# (csrc/consensus.h: SparqArgs).  A node whose tail says 0 is not pulled past its tail.
SPARQ_COMPRESSORS = ("none", "int8", "sign")
SPARQ_TAIL = 16


def sparq_row_bytes(code_bytes: int) -> int:
    """Bytes of one published SPARQ row: the code row and the tail, rounded up to 16."""
    return -(-(int(code_bytes) + SPARQ_TAIL) // 16) * 16


def sparq_threshold(threshold: float, growth: float, alphas) -> np.ndarray:
    """``thr_k = threshold (k + 1)^growth alpha_k^2`` in float64 for the given ``alpha_k`` of rounds 0, 1, ..."""
    a = np.asarray(alphas, dtype=np.float64)
    k1 = np.arange(1, a.size + 1, dtype=np.float64)
    return float(threshold) * k1 ** float(growth) * (a * a)


def sparq_tails(trig: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """``[L, 16]`` uint8 tails of trigger bits ``trig [L]`` and errors ``e [L]`` (float64)."""
    L = trig.shape[0]
    head = torch.stack([trig.to(torch.int32), torch.zeros_like(trig, dtype=torch.int32)], dim=1).contiguous()
    return torch.cat([head.view(torch.uint8).reshape(L, 8),
                      e.to(torch.float64).reshape(L, 1).contiguous().view(torch.uint8).reshape(L, 8)], dim=1)


def sparq_tail_read(rows: torch.Tensor, code_bytes: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The trigger bits (bool ``[R]``) and errors (float64 ``[R]``) in the tails of published rows ``[R, row_bytes]``."""
    t = rows[:, code_bytes: code_bytes + SPARQ_TAIL].contiguous()
    return t[:, :4].view(torch.int32)[:, 0] != 0, t[:, 8:].view(torch.float64)[:, 0]


def sparq_mix_(theta: torch.Tensor, x_hat: torch.Tensor, s: torch.Tensor, rows_all: torch.Tensor, w_rows: torch.Tensor,
               gamma: float, compressor: str, live: torch.Tensor, code_bytes: int) -> None:
    """``s_i += sum_j W_ij dec(q_j)`` over the nodes whose pending tail says triggered (own term included), then
    ``theta_i += gamma (s_i - x_hat_i)``.  A non-triggered row's body is not decoded into the sum (it may be stale)."""
    trig, _ = sparq_tail_read(rows_all, code_bytes)
    dec = choco_decode(rows_all[:, :code_bytes], compressor, theta.shape[1], theta.dtype, live)
    dec = torch.where(trig.to(dec.device)[:, None], dec, torch.zeros((), dtype=dec.dtype, device=dec.device))
    choco_mix_(theta, x_hat, s, dec, w_rows, gamma)


def sparq_step_(theta: torch.Tensor, grad: torch.Tensor, alpha: float) -> None:
    """One local step ``theta -= alpha g`` (DSGD's)."""
    theta.add_(grad, alpha=-alpha)


def sparq_publish_(theta: torch.Tensor, x_hat: torch.Tensor, code: torch.Tensor, thr: float, compressor: str,
                   live: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``e_i = ||theta_i - x_hat_i||^2`` (float64), ``trig_i = e_i > thr``.  A triggered node writes ``Q(theta_i -
    x_hat_i)`` into the body of its row ``code [L, row_bytes]`` and takes ``x_hat_i += dec``; every node writes its tail.
    Returns ``(trig, e)``."""
    v = theta - x_hat
    e = (v.to(torch.float64) ** 2).sum(1)
    trig = e > float(thr)
    codes, dec = choco_encode(v, compressor, live)
    cb = codes.shape[1]
    code[:, :cb] = torch.where(trig[:, None], codes, code[:, :cb])
    x_hat.copy_(torch.where(trig[:, None], x_hat + dec, x_hat))
    code[:, cb: cb + SPARQ_TAIL] = sparq_tails(trig, e)
    return trig, e


# ----------------------------------------------------------------- BEER ----
# Gradient tracking with both channels gossiped as CHOCO codes: channel 0 codes theta - h, channel 1 codes v - g, with
# CHOCO's encoder, decoder and byte layout.
def beer_mix_(theta: torch.Tensor, h: torch.Tensor, s_h: torch.Tensor, v: torch.Tensor, s_g: torch.Tensor,
              dec_h_all: torch.Tensor, dec_g_all: torch.Tensor, w_rows: torch.Tensor, gamma: float, alpha: float):
    """``s_h_i += sum_j W_ij dec(qh_j)``, ``s_g_i += sum_j W_ij dec(qg_j)`` (own terms included);
    ``theta_i += gamma (s_h_i - h_i) - alpha v_i``."""
    w = w_rows.to(dec_h_all.dtype)
    s_h.add_(w @ dec_h_all)
    s_g.add_(w @ dec_g_all)
    theta.add_(gamma * (s_h - h) - alpha * v)


def beer_step_(theta: torch.Tensor, h: torch.Tensor, v: torch.Tensor, g: torch.Tensor, s_g: torch.Tensor,
               m_old: torch.Tensor, grad: torch.Tensor, gamma: float, compressor: str,
               live: torch.Tensor, k: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """``v += gamma (s_g - g) + grad - m_old``; ``m_old <- grad``; ``qh = Q(theta - h)``, ``h += dec(qh)``;
    ``qg = Q(v - g)``, ``g += dec(qg)``; returns the code rows ``(qh, qg)`` to publish."""
    v.add_(gamma * (s_g - g) + grad - m_old)
    m_old.copy_(grad)
    codes_h, dec_h = choco_encode(theta - h, compressor, live, k)
    h.add_(dec_h)
    codes_g, dec_g = choco_encode(v - g, compressor, live, k)
    g.add_(dec_g)
    return codes_h, codes_g


# ----------------------------------------------------------------- K-GT ----
def kgt_mix_(theta: torch.Tensor, c: Optional[torch.Tensor], theta_all: torch.Tensor, y_all: Optional[torch.Tensor],
             y: Optional[torch.Tensor], w_rows: torch.Tensor):
    """``theta_i <- sum_j W_ij theta_j``; with a correction row ``c`` also ``c_i += sum_j W_ij y_j - y_i`` (own terms
    included).  Without it this is DSGD's mix."""
    theta.copy_(dsgd_mix(theta_all, w_rows))
    if c is not None:
        c.add_(dsgd_mix(y_all, w_rows) - y)


def kgt_step_(theta: torch.Tensor, c: Optional[torch.Tensor], d: Optional[torch.Tensor], grad: torch.Tensor,
              alpha: float, p: int, K: int) -> Optional[torch.Tensor]:
    """Local step ``p`` of ``K``: ``u = g + c`` (``g`` without ``c``), ``theta -= alpha u``, ``d = u`` (p = 0) or
    ``d += u``.  Returns ``y = d / K`` on the last step with a correction row, else ``None``.  Without ``c`` this is
    DSGD's step."""
    if c is None:
        dsgd_step_(theta, grad, alpha)
        return None
    u = grad + c
    theta.sub_(alpha * u)
    if p == 0:
        d.copy_(u)
    else:
        d.add_(u)
    return d / K if p == K - 1 else None


# ------------------------------------------------- decentralized adaptive ----
DADAPTIVE_VARIANTS = ("amsgrad", "adagrad")


def dadaptive_mix_(theta: torch.Tensor, ut: Optional[torch.Tensor], theta_all: torch.Tensor,
                   ut_all: Optional[torch.Tensor], w_rows: torch.Tensor):
    """``x_i = sum_j W_ij theta_j`` into ``theta``; with tracking also ``z_i = sum_j W_ij u~_j`` into ``ut`` (the row
    holds z until the step turns it into the new tracker).  Without tracking this is DSGD's mix."""
    theta.copy_(dsgd_mix(theta_all, w_rows))
    if ut is not None:
        ut.copy_(dsgd_mix(ut_all, w_rows))


def dadaptive_step_(theta: torch.Tensor, m: torch.Tensor, v: Optional[torch.Tensor], vhat: torch.Tensor,
                    ut: Optional[torch.Tensor], grad: torch.Tensor, alpha: float, beta1: float, beta2: float,
                    eps: float, k: int, adagrad: bool):
    """The adaptive step of round ``k`` on the mixed rows ``x = theta`` (``ut`` holds z of the mix, or is ``None``
    without tracking):

        m <- beta1 m + (1 - beta1) g
        amsgrad:  v <- beta2 v + (1 - beta2) g^2;  vhat' = max(vhat, v)
        adagrad:  vhat' = vhat + (g^2 - vhat) / (k + 1)
        tracking: u~ <- z + (vhat' - vhat);  u = max(u~, eps)      own: u = max(vhat', eps)
        vhat <- vhat';  theta <- x - alpha m / sqrt(u)"""
    m.mul_(beta1).add_(grad, alpha=1.0 - beta1)
    g2 = grad * grad
    if adagrad:
        vn = vhat + (g2 - vhat) / float(k + 1)
    else:
        v.mul_(beta2).add_(g2, alpha=1.0 - beta2)
        vn = torch.maximum(vhat, v)
    if ut is not None:
        ut.add_(vn - vhat)
        u = ut.clamp_min(eps)
    else:
        u = vn.clamp_min(eps)
    vhat.copy_(vn)
    theta.sub_(alpha * (m / u.sqrt()))


# --------------------------------------------------------------- RelaySum ----
def relaysum_mix_(theta: torch.Tensor, msg_all: List[torch.Tensor], src_node: torch.Tensor, src_slot: torch.Tensor,
                  live: torch.Tensor, reach_m1: torch.Tensor, n: int) -> torch.Tensor:
    """The mix of round k for the local rows ``theta`` (holding h): ``r_e = m_{j_e -> i}``, gathered from
    ``msg_all[s]`` (every node's published message slot s, ``[N, n_pad]``) at ``[src_slot, src_node]`` (``[L, dmax]``,
    the neighbor j_e and its reverse slot; ``live`` marks e < deg_i), then ``x = h + (sum_e r_e - (R_i^k - 1) h) / n``
    with e ascending (``reach_m1``: ``[L]``).  Returns ``r`` (``[L, dmax, n_pad]``, zero past deg_i) for the step."""
    r = torch.stack(msg_all)[src_slot, src_node]
    r = torch.where(live[:, :, None], r, torch.zeros((), dtype=r.dtype))
    s = torch.zeros_like(theta)
    for e in range(r.shape[1]):
        s = s + r[:, e]
    theta.copy_(theta + (s - reach_m1[:, None] * theta) / n)
    return r


def relaysum_step_(theta: torch.Tensor, msg: torch.Tensor, r: torch.Tensor, live: torch.Tensor, grad: torch.Tensor,
                   alpha: float):
    """``h = x - alpha g`` into ``theta``, and the messages ``m_{i -> j_e} = h + sum_{e' != e} r_e'`` (e' ascending)
    into ``msg[:, e]`` (``[L, dmax, n_pad]``; zero past deg_i)."""
    theta.add_(grad, alpha=-alpha)
    for e in range(msg.shape[1]):
        m = theta.clone()
        for f in range(r.shape[1]):
            if f != e:
                m = m + r[:, f]
        msg[:, e] = torch.where(live[:, e, None], m, torch.zeros((), dtype=m.dtype))


# ------------------------------------------------------------- PowerGossip ----
class PgLayout:
    """The matrix table of PowerGossip, from a ``FlatLayout``: every parameter tensor with two or more dimensions is a
    matrix ``(shape[0], prod(shape[1:]))``, the others (biases) are gossiped whole.  In slot order, ``segs`` holds one
    ``(offset, m, n, poff, qoff)`` per tensor: for a matrix ``poff`` / ``qoff`` are its offsets in the row space
    (``P = sum m``) and the column space (``Q = sum n``); for a 1-D tensor ``n = 0``, ``m`` is its length and ``poff``
    its offset in the bias block (``B`` elements).  A phase-0 message is ``[the products h q (P) | biases (B)]``, a
    phase-1 message ``[h^T p (Q) | biases (B)]``; ``width`` is the longer of the two, rounded up to 16 bytes in either
    dtype (consensus.h: PgArgs)."""

    def __init__(self, layout):
        self.segs: List[Tuple[int, int, int, int, int]] = []
        P = Q = B = 0
        for s in layout.slots:
            if len(s.shape) >= 2:
                m = int(s.shape[0])
                n = int(s.numel) // m
                self.segs.append((int(s.offset), m, n, P, Q))
                P += m
                Q += n
            else:
                self.segs.append((int(s.offset), int(s.numel), 0, B, 0))
                B += int(s.numel)
        self.P, self.Q, self.B = P, Q, B
        self.mats = [sg for sg in self.segs if sg[2] > 0]
        self.vecs = [sg for sg in self.segs if sg[2] == 0]
        self.width = -(-max(P + B, Q + B, 1) // 4) * 4

    def msg_len(self, phase: int) -> int:
        """Elements of a message of ``phase`` (unpadded)."""
        return (self.Q if phase else self.P) + self.B


def pg_start_vectors(lay: PgLayout, lo: int, hi: int, dtype: torch.dtype) -> torch.Tensor:
    """``[P + Q]``: the unit vectors ``p_{e,l}`` (row space) then ``q_{e,l}`` (column space) of edge ``{lo, hi}``
    (``lo < hi``), drawn for matrix l from ``np.random.default_rng((lo, hi, l))`` (p first), normalised in float64 and
    rounded once to ``dtype``.  Both endpoints draw the same vectors."""
    out = np.zeros(lay.P + lay.Q)
    for l, (_, m, n, poff, qoff) in enumerate(lay.mats):
        rng = np.random.default_rng((lo, hi, l))
        p = rng.standard_normal(m)
        q = rng.standard_normal(n)
        out[poff: poff + m] = p / np.linalg.norm(p)
        out[lay.P + qoff: lay.P + qoff + n] = q / np.linalg.norm(q)
    return torch.as_tensor(out).to(dtype)


def pg_sumsq(d: torch.Tensor) -> torch.Tensor:
    """``sum d^2`` over the last dimension in float64, in the order of one warp of pg_mix_kernel: lane t sums the
    elements t, t + 32, ... (each square rounded, then added), then the 32 lane sums are combined by xor butterflies
    16, 8, 4, 2, 1.  Bit for bit the kernel's value, whatever the row's position in a batch."""
    x = d.double()
    n = x.shape[-1]
    x = torch.nn.functional.pad(x, (0, (-n) % 32)).reshape(*x.shape[:-1], -1, 32)
    s = torch.zeros(x.shape[:-2] + (32,), dtype=torch.float64, device=x.device)
    for c in range(x.shape[-2]):
        s = s + x[..., c, :] * x[..., c, :]
    lane = torch.arange(32, device=x.device)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    return s[..., 0]


def pg_messages(h: torch.Tensor, vec: torch.Tensor, live: torch.Tensor, lay: PgLayout, phase: int) -> torch.Tensor:
    """The messages ``[L, dmax, width]`` node i publishes for its neighbor slots after its step: per matrix the product
    ``h q_e`` (phase 0, length m) or ``h^T p_e`` (phase 1, length n), then h's 1-D tensors; zero past deg_i and past the
    phase's length."""
    L, dmax = live.shape
    msg = torch.zeros(L, dmax, lay.width, dtype=h.dtype, device=h.device)
    for off, m, n, poff, qoff in lay.mats:
        H = h[:, off: off + m * n].reshape(L, 1, m, n)
        if phase == 0:
            q = vec[:, :, lay.P + qoff: lay.P + qoff + n]
            msg[:, :, poff: poff + m] = (H @ q[..., None])[..., 0]
        else:
            p = vec[:, :, poff: poff + m]
            msg[:, :, qoff: qoff + n] = (p[:, :, None, :] @ H)[:, :, 0]
    base = lay.Q if phase else lay.P
    for off, m, _, boff, _ in lay.vecs:
        msg[:, :, base + boff: base + boff + m] = h[:, None, off: off + m]
    return torch.where(live[:, :, None], msg, torch.zeros((), dtype=msg.dtype))


def pg_mix_(theta: torch.Tensor, vec: torch.Tensor, own: torch.Tensor, nbr: torch.Tensor, sign: torch.Tensor,
            w: torch.Tensor, live: torch.Tensor, gamma: float, lay: PgLayout, phase: int):
    """The mix of round k (``phase = k & 1``) for the local rows ``theta`` (holding h).  ``own`` / ``nbr``
    (``[L, dmax, width]``) are the messages node i and its neighbor j_e published for edge e; ``sign`` is +1 where
    i < j_e, else -1.  Per edge, ``d = a_lo - a_hi`` (the same bits at both endpoints), ``U_e = d q^T`` (phase 0) or
    ``p d^T`` (phase 1) per matrix and the whole difference for the 1-D tensors; then
    ``x = h - gamma * sum_e (W_ie s_ie) U_e`` (e ascending) into ``theta``.  The next vectors ``p <- d / |d|``
    (phase 0) or ``q <- d / |d|`` (phase 1) go into ``vec``, with ``|d|`` from ``pg_sumsq`` and one rounding; a zero
    difference keeps the stored vector."""
    L, dmax = live.shape
    d = torch.where(sign[:, :, None] > 0, own - nbr, nbr - own)
    coef = w * sign.to(w.dtype)
    acc = torch.zeros_like(theta)
    for off, m, n, poff, qoff in lay.mats:
        a = torch.zeros(L, m, n, dtype=theta.dtype, device=theta.device)
        for e in range(dmax):
            if phase == 0:
                U = d[:, e, poff: poff + m, None] * vec[:, e, None, lay.P + qoff: lay.P + qoff + n]
            else:
                U = vec[:, e, poff: poff + m, None] * d[:, e, None, qoff: qoff + n]
            a = torch.where(live[:, e, None, None], a + coef[:, e, None, None] * U, a)
        acc[:, off: off + m * n] = a.reshape(L, m * n)
    base = lay.Q if phase else lay.P
    for off, m, _, boff, _ in lay.vecs:
        a = torch.zeros(L, m, dtype=theta.dtype, device=theta.device)
        for e in range(dmax):
            U = d[:, e, base + boff: base + boff + m]
            a = torch.where(live[:, e, None], a + coef[:, e, None] * U, a)
        acc[:, off: off + m] = a
    theta.sub_(gamma * acc)
    for off, m, n, poff, qoff in lay.mats:
        lo, ln = (poff, m) if phase == 0 else (qoff, n)
        out = poff if phase == 0 else lay.P + qoff
        dl = d[:, :, lo: lo + ln]
        ss = pg_sumsq(dl)
        keep = (ss == 0) | ~live
        nv = (dl.double() / ss.sqrt()[..., None]).to(vec.dtype)
        vec[:, :, out: out + ln] = torch.where(keep[..., None], vec[:, :, out: out + ln], nv)


def pg_step_(theta: torch.Tensor, msg: torch.Tensor, grad: torch.Tensor, alpha: float, vec: torch.Tensor,
             live: torch.Tensor, lay: PgLayout, phase: int):
    """``h = x - alpha g`` into ``theta``, and the messages of ``phase`` (that of round k + 1) into ``msg``."""
    theta.add_(grad, alpha=-alpha)
    msg.copy_(pg_messages(theta, vec, live, lay, phase))


# ---------------------------------------------------------- ClippedGossip ----
ATTACK_CODE = {"sign_flip": 1, "alie": 2}      # consensus.h: Attack (0 = honest)
CLIP_SLACK = 1e-6      # consensus.h: kClipSlack, a prefix of (rounded) weights fits in delta up to this


def cg_distances(theta_i: torch.Tensor, nbr_rows: torch.Tensor) -> np.ndarray:
    """``d_ij = |theta_j^pub - theta_i|_2`` of every neighbor row (``nbr_rows`` [deg, n_pad]), accumulated in fp64."""
    if nbr_rows.shape[0] == 0:
        return np.zeros(0)
    diff = nbr_rows.double() - theta_i.double()
    return (diff * diff).sum(1).sqrt().cpu().numpy()


def cg_factors(d: np.ndarray, w: np.ndarray, delta: float) -> Tuple[np.ndarray, float]:
    """Radius and clipping factors of one node: the neighbors in order of decreasing distance (ties: the smaller index
    first) are clipped while their Metropolis weights ``w`` sum to at most ``delta`` (up to ``CLIP_SLACK``); ``tau`` is the distance of the
    first one that does not fit (0 when all fit) and the factor of edge j is ``min(1, tau / d_ij)`` (1 at d_ij = 0)."""
    order = sorted(range(len(d)), key=lambda e: (-d[e], e))
    cum, tau = 0.0, 0.0
    for e in order:
        if cum + float(w[e]) > delta + CLIP_SLACK:
            tau = float(d[e])
            break
        cum += float(w[e])
    f = np.array([tau / d[e] if d[e] > tau else 1.0 for e in range(len(d))])
    return f, tau


def cg_mix_(theta: torch.Tensor, pub_all: torch.Tensor, w_rows: np.ndarray, nbrs, lo: int, delta: float):
    """Self-centred clipped mix of the local rows ``theta`` [L, n_pad]:
    ``theta_i <- theta_i + sum_j W_ij min(1, tau_i / d_ij) (theta_j^pub - theta_i)``, in neighbor order, the
    coefficient ``W_ij * factor`` rounded to the row dtype once (as cg_mix_kernel).  ``pub_all`` [N, n_pad] holds every
    node's published row, ``w_rows`` the Metropolis matrix (host, rounded to the row dtype), ``nbrs[g]`` the neighbors
    of node g in table order.  Returns the factors of every local node."""
    out = []
    for l in range(theta.shape[0]):
        nb = list(nbrs[lo + l])
        th0 = theta[l].clone()
        rows = pub_all[nb] if nb else pub_all[:0]
        w = np.array([float(w_rows[lo + l, j]) for j in nb])
        f, _ = cg_factors(cg_distances(th0, rows), w, delta)
        acc = th0.clone()
        for e in range(len(nb)):
            coef = torch.tensor(w[e] * f[e], dtype=theta.dtype)
            acc += coef * (rows[e] - th0)
        theta[l].copy_(acc)
        out.append(f)
    return out


def cg_publish_(pub: torch.Tensor, theta: torch.Tensor, pub_all: torch.Tensor, attack, nbrs, byz, lo: int,
                scale: float, z: float):
    """Write into ``pub`` [L, n_pad] the rows the local nodes publish after their step.  ``attack[l]``: 0 honest (theta), 1 sign flip
    (``-scale theta``), 2 ALIE (``mu - z sigma``, the fp64 element-wise mean and population standard deviation of the
    node's honest neighbors' rows in ``pub_all``, the rows read this round; theta without an honest neighbor)."""
    out = theta.clone()          # pub_all may alias pub (one process holds every row)
    s = torch.tensor(scale, dtype=theta.dtype)
    for l, code in enumerate(attack):
        if code == 1:
            out[l] = -(s * theta[l])
        elif code == 2:
            hon = [j for j in nbrs[lo + l] if j not in byz]
            if hon:
                x = pub_all[hon].double()
                mu = x.mean(0)
                sigma = ((x - mu) ** 2).mean(0).sqrt()
                out[l] = (mu - z * sigma).to(theta.dtype)
    pub.copy_(out)


# ----------------------------------------------------------------- BRIDGE ----
BRIDGE_SCREENS = ("trimmed_mean", "median")


def bridge_mix_(theta: torch.Tensor, pub_all: torch.Tensor, nbrs, lo: int, screen: str, b: int = 0):
    """Coordinate-wise screened mix of the local rows ``theta`` [L, n_pad] (bridge_mix_kernel): per element, the
    neighbors' values of ``pub_all`` [N, n_pad] sorted (``torch.sort`` over the neighbor axis), then
    ``trimmed_mean``: ``(theta_i + sorted positions [b, deg - b) in ascending order) / (1 + max(0, deg - 2b))``, or
    ``median``: the median of theta_i and the deg values (``0.5 (lower + upper)`` of an even count), in fp64 and rounded
    once to the row dtype.  ``nbrs[g]``: the neighbors of node g."""
    out = theta.clone()
    for l in range(theta.shape[0]):
        nb = list(nbrs[lo + l])
        x = theta[l].double()
        s = torch.sort(pub_all[nb].double(), dim=0).values if nb else pub_all[:0].double()
        deg = len(nb)
        if screen == "median":
            allv = torch.sort(torch.cat([x[None], s]), dim=0).values
            y = allv[deg // 2] if deg % 2 == 0 else 0.5 * (allv[deg // 2] + allv[deg // 2 + 1])
        else:
            acc = x.clone()
            for p in range(b, deg - b):
                acc = acc + s[p]
            y = acc / (1 + max(0, deg - 2 * b))
        out[l] = y.to(theta.dtype)
    theta.copy_(out)


# ------------------------------------------------------------------ SGP ----
# Push-sum (Stochastic Gradient Push): numerator rows x [L, n_pad] and float64 weights w [L].  The combine weights are
# the column-stochastic A of Topology.push_weights, rounded to the arena dtype; w is mixed with those same rounded
# weights (in float64), so x and w see one matrix.
def sgp_debias(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """``theta = x / w``: w rounded to x's dtype, then one IEEE division in that dtype (csrc: sgp_debias)."""
    return x / w.to(x.dtype).unsqueeze(1)


def sgp_mix_(x: torch.Tensor, w: torch.Tensor, theta: torch.Tensor, x_all: torch.Tensor, w_all: torch.Tensor,
             a_rows: torch.Tensor):
    """``x_i <- sum_j A_ij x_j``, ``w_i <- sum_j A_ij w_j`` (own term included), ``theta_i <- x_i / w_i``."""
    a = a_rows.to(x_all.dtype)
    x.copy_(a @ x_all)
    w.copy_(a.to(torch.float64) @ w_all.to(torch.float64))
    theta.copy_(sgp_debias(x, w))


def sgp_step_(x: torch.Tensor, w: torch.Tensor, theta: torch.Tensor, grad: torch.Tensor, alpha: float):
    """``x <- x - alpha g`` (g taken at theta = x / w); ``theta <- x / w``."""
    x.add_(grad, alpha=-alpha)
    theta.copy_(sgp_debias(x, w))


# ---------------------------------------------------------- Push-DIGing ----
# Gradient tracking on push-sum gossip: numerators u [L, n_pad], float64 weights w [L], trackers y [L, n_pad].  SGP's
# rounding rules: the weights of A rounded to the arena dtype, w mixed in float64 with those rounded weights, and
# theta = u / w by sgp_debias.
def pdg_mix_(u: torch.Tensor, w: torch.Tensor, theta: torch.Tensor, ysum: torch.Tensor, u_all: torch.Tensor,
             y_all: torch.Tensor, w_all: torch.Tensor, a_rows: torch.Tensor, alpha: float):
    """``u_i <- sum_j A_ij (u_j - alpha y_j)``, ``ysum_i <- sum_j A_ij y_j``, ``w_i <- sum_j A_ij w_j`` (own terms
    included), ``theta_i <- u_i / w_i``."""
    a = a_rows.to(u_all.dtype)
    u.copy_(a @ (u_all - alpha * y_all))
    ysum.copy_(a @ y_all)
    w.copy_(a.to(torch.float64) @ w_all.to(torch.float64))
    theta.copy_(sgp_debias(u, w))


def pdg_track_(y: torch.Tensor, g_old: torch.Tensor, ysum: torch.Tensor, grad: torch.Tensor):
    """``y <- ysum + (g - g_old)``, ``g_old <- g`` (g taken at theta = u / w)."""
    y.copy_(ysum + (grad - g_old))
    g_old.copy_(grad)


# ---------------------------------------------------------------- DP-DSGD ----
# The noise stream (consensus.h: DpArgs): Philox4x32-10, key (lo32(seed), hi32(seed) ^ DP_KEY_DOMAIN), counter
# (element pair p, round k, a, b) with (a, b) = (i, DP_LOCAL) for node i's own stream and (min(i, j), max(i, j)) for
# edge {i, j}.  One call gives the normals of elements 2p and 2p + 1 by Box-Muller in float64.
DP_KEY_DOMAIN = 0x44505347          # "DPSG": the DP key never equals the problem seed's plain Philox key
DP_LOCAL = 0xFFFFFFFF               # b of a node's own stream (no node id is 2^32 - 1)
_PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC 2011; curand's ``curand_Philox4x32_10``) of the counters
    ``ctr [..., 4]`` under ``key (k0, k1)``, vectorised over the leading axes: ``[..., 4]`` uint32."""
    c = [np.asarray(x, dtype=np.uint64) & _M32 for x in np.moveaxis(np.asarray(ctr, dtype=np.uint64), -1, 0)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + _PHILOX_W[0]) & 0xFFFFFFFF, (k1 + _PHILOX_W[1]) & 0xFFFFFFFF
        p0, p1 = _PHILOX_M[0] * c[0], _PHILOX_M[1] * c[2]       # exact: 32 x 32 bits in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1),
             p0 & _M32]
    return np.stack(c, axis=-1).astype(np.uint32)


def dp_key(seed: int) -> Tuple[int, int]:
    """The 64-bit Philox key of the DP noise for ``noise_seed`` (any integer, taken mod 2^64)."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, (s >> 32) ^ DP_KEY_DOMAIN


def _cospi_sinpi(x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """``(cos(pi x), sin(pi x))`` for x in [0, 2) a multiple of 2^-52: x = q / 2 + y exactly with |y| <= 1/4, so the
    rounding of ``pi y`` stays below 1e-16 absolute."""
    q = np.rint(2.0 * x)
    y = x - 0.5 * q
    c, s = np.cos(np.pi * y), np.sin(np.pi * y)
    q = q.astype(np.int64) & 3
    cs = np.select([q == 0, q == 1, q == 2], [c, -s, -c], s)
    sn = np.select([q == 0, q == 1, q == 2], [s, c, -s], -c)
    return cs, sn


def dp_normals(key, k: int, a: int, b: int, n_pad: int) -> np.ndarray:
    """The ``[n_pad]`` float64 standard normals of stream ``(a, b)`` in round k (before the live mask)."""
    p = np.arange(n_pad // 2, dtype=np.uint64)
    ctr = np.stack([p, np.full_like(p, k), np.full_like(p, a), np.full_like(p, b)], axis=-1)
    x = philox4x32_10(ctr, key).astype(np.uint64)
    u1 = (((x[:, 0] >> np.uint64(5)) << np.uint64(26)) + (x[:, 1] >> np.uint64(6)) + np.uint64(1)).astype(np.float64)
    u2 = (((x[:, 2] >> np.uint64(5)) << np.uint64(26)) + (x[:, 3] >> np.uint64(6))).astype(np.float64)
    u1 *= 2.0 ** -53
    u2 *= 2.0 ** -53
    r = np.sqrt(-2.0 * np.log(u1))
    c, s = _cospi_sinpi(2.0 * u2)
    out = np.empty(n_pad)
    out[0::2], out[1::2] = r * c, r * s
    return out


def dp_noise(key, k: int, i: int, nbrs, n_pad: int, cz_dp: float, cz_pair: float, live: np.ndarray) -> np.ndarray:
    """``v_i`` of round k in float64 (``[n_pad]``, 0 off the live elements): ``cz_dp xi_i + cz_pair sum_j s_ij xi_ij``
    over the neighbors ``nbrs`` in table order, ``s_ij = +1`` if i < j else -1, with ``cz = C z`` rounded once.  The
    kernel (dp_step_kernel) evaluates the same expression in the same order."""
    v = np.zeros(n_pad)
    if cz_dp != 0.0:
        v = cz_dp * dp_normals(key, k, i, DP_LOCAL, n_pad)
    if cz_pair != 0.0 and len(nbrs):
        e = np.zeros(n_pad)
        for j in nbrs:
            xi = dp_normals(key, k, min(i, j), max(i, j), n_pad)
            e = e + xi if i < j else e - xi
        v = v + cz_pair * e
    return np.where(live, v, 0.0)


def dp_clip_factor(sumsq: float, clip: float) -> float:
    """``min(1, C / ||g||)`` from ``||g||^2`` in float64 (1 when g = 0)."""
    nrm = math.sqrt(sumsq)
    return clip / nrm if nrm > clip else 1.0


def dp_rho(W: np.ndarray, z_dp: float, z_pair: float) -> Tuple[np.ndarray, np.ndarray]:
    """zCDP cost ``[N]`` of one round per node, (eavesdropper, any observer) (DESIGN §2.16): the noise of one coordinate
    across nodes has covariance ``C^2 Sigma``, ``Sigma = z_dp^2 I + z_pair^2 Lap(G)``; replacing node i's shard moves
    its row by at most ``2 C alpha``, so rho = 2 [Sigma^-1]_ii for an observer who sees every published row and knows no
    pair secret, and 2 / z_dp^2 for one who knows them all.  ``W`` only gives the graph (its off-diagonal support)."""
    N = W.shape[0]
    if z_dp == 0.0:
        inf = np.full(N, np.inf)
        return inf, inf.copy()
    A = ((W != 0) & ~np.eye(N, dtype=bool)).astype(np.float64)
    lap = np.diag(A.sum(1)) - A
    sigma = z_dp * z_dp * np.eye(N) + z_pair * z_pair * lap
    return 2.0 * np.diag(np.linalg.inv(sigma)).copy(), np.full(N, 2.0 / (z_dp * z_dp))


def dp_epsilon(rho, delta: float) -> float:
    """(epsilon, delta)-DP of a rho-zCDP ledger, ``rho + 2 sqrt(rho ln(1/delta))``, the maximum over its nodes."""
    rho = np.asarray(rho, dtype=np.float64)
    return float(np.max(rho + 2.0 * np.sqrt(rho * math.log(1.0 / delta))))


# ---------------------------------------------------------------- Moniqua ----
# Code rows (the layout of csrc/consensus.h: MoniquaArgs, the only other place it is written): b-bit codes of the
# parameters modulo the range B, element e at bit (e b) % 32 of 32-bit word (e b) / 32, little-end first, so a row
# is n_pad b / 8 bytes.  With L = 2^b and delta = 1 / L, all in float64:
#   encode  t = frac(x / B) L;  c = (floor(t) + (u < t - floor(t))) mod L     u from the rounding stream
#   decode  v = y / B - c / L;  n = rint(v);  xhat = B (c / L + n);  margin offset v - n   (y: the reader's own value)
# The rounding stream is Philox4x32-10 under mq_key(rounding_seed) with the counter (e / 4, k, node, MQ_TAG): output
# word e % 4 gives u = r 2^-32 for element e of the code that `node` publishes for round k (read in round k).  Padding
# and slot holes get code 0.  Every division and product is a single IEEE operation, so the kernels write the same bits.
MQ_BITS = (2, 4, 8)
MQ_BASES = ("dsgd", "exact_diffusion")
MQ_KEY_DOMAIN = 0x4D4E5155          # "MNQU": the rounding key never equals the problem seed's plain Philox key
MQ_TAG = 0x4D515244                 # "MQRD": the fourth counter word of the rounding stream


def mq_key(seed: int) -> Tuple[int, int]:
    """The 64-bit Philox key of the rounding stream for ``rounding_seed`` (any integer, taken mod 2^64)."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, (s >> 32) ^ MQ_KEY_DOMAIN


def mq_range(theta_bound: float, bits: int) -> float:
    """``B = 2 theta_bound / (1 - 2 delta)``, ``delta = 2^-bits``: the modulus that makes every decode exact while the
    reader is within ``theta_bound`` of the value behind the code (DESIGN §2.17)."""
    return 2.0 * float(theta_bound) / (1.0 - 2.0 * 2.0 ** -int(bits))


def mq_code_bytes(n_pad: int, bits: int) -> int:
    """Bytes of one code row; rows must be padded to a multiple of 128 elements, so rows stay 16-byte aligned."""
    if n_pad % 128 != 0:
        raise ValueError(f"moniqua needs rows padded to a multiple of 128 elements (n_pad = {n_pad})")
    return n_pad * int(bits) // 8


def mq_uniforms(key, k: int, node: int, n_pad: int) -> np.ndarray:
    """The ``[n_pad]`` float64 uniforms ``r 2^-32`` that round the code ``node`` publishes for round ``k``."""
    p = np.arange(n_pad // 4, dtype=np.uint64)
    ctr = np.stack([p, np.full_like(p, k), np.full_like(p, node), np.full_like(p, MQ_TAG)], axis=-1)
    return philox4x32_10(ctr, key).reshape(-1).astype(np.float64) * 2.0 ** -32


def mq_codes(x: torch.Tensor, B: float, bits: int, u: torch.Tensor, live: torch.Tensor) -> torch.Tensor:
    """The codes ``[R, n_pad]`` (int64, in ``[0, 2^bits)``) of the rows ``x`` with the uniforms ``u`` (same shape)."""
    L = 1 << bits
    z = x.double() / B
    t = (z - torch.floor(z)) * L
    fl = torch.floor(t)
    c = (fl.to(torch.int64) + (u.to(t.device) < t - fl).to(torch.int64)) % L
    return torch.where(live.to(c.device), c, torch.zeros_like(c))


def mq_pack(codes: torch.Tensor, bits: int) -> torch.Tensor:
    """Code rows ``[R, n_pad b / 8]`` (uint8) of the codes ``[R, n_pad]``."""
    R, n_pad = codes.shape
    per = 32 // bits
    shifts = torch.arange(per, device=codes.device, dtype=torch.int64) * bits
    words = (codes.reshape(R, n_pad // per, per) << shifts).sum(-1)
    return torch.stack([(words >> (8 * q)) & 255 for q in range(4)], dim=-1).to(torch.uint8).reshape(R, -1)


def mq_unpack(rows: torch.Tensor, bits: int) -> torch.Tensor:
    """The codes ``[R, n_pad]`` (int64) of code rows ``[R, n_pad b / 8]`` (uint8)."""
    R = rows.shape[0]
    wb = rows.to(torch.int64).reshape(R, -1, 4)
    words = wb[..., 0] | (wb[..., 1] << 8) | (wb[..., 2] << 16) | (wb[..., 3] << 24)
    per = 32 // bits
    shifts = torch.arange(per, device=rows.device, dtype=torch.int64) * bits
    return ((words.unsqueeze(-1) >> shifts) & ((1 << bits) - 1)).reshape(R, -1)


def mq_encode(x: torch.Tensor, B: float, bits: int, key, k: int, nodes, live: torch.Tensor) -> torch.Tensor:
    """Code rows ``[R, n_pad b / 8]`` (uint8) that the nodes ``nodes`` (global ids, one per row of ``x``) publish for
    round ``k``."""
    u = torch.as_tensor(np.stack([mq_uniforms(key, k, int(g), x.shape[1]) for g in nodes]), device=x.device)
    return mq_pack(mq_codes(x, B, bits, u, live), bits)


def mq_decode(codes: torch.Tensor, y: torch.Tensor, B: float, bits: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(xhat, v - n)`` in float64 of the codes ``codes`` (int64) decoded against the side information ``y``."""
    cl = codes.double() * 2.0 ** -bits
    v = y.double() / B - cl
    n = torch.round(v)                     # half to even, as rint
    return B * (cl + n), v - n


def mq_margin_hits(off: torch.Tensor, bits: int) -> torch.Tensor:
    """Margin hits: elements whose decode offset is past ``1/2 - delta`` (at or near the wrap boundary)."""
    return off.abs() > 0.5 - 2.0 ** -bits


def mq_mix_(theta: torch.Tensor, codes_all: torch.Tensor, w_rows: torch.Tensor, nbrs, lo: int, B: float, bits: int,
            margin: torch.Tensor) -> None:
    """The combine of the local rows: ``theta_i += sum_{j != i} w_ij (xhat_j - xhat_i)``, every code decoded against
    ``y = theta_i``, the sum in float64 over the neighbors ``nbrs[l]`` (global ids) in table order with the weights of
    ``w_rows [L, N]`` (in the arena dtype), rounded once.  ``codes_all [N, n_pad]`` are every node's pending codes;
    each neighbor element past the margin adds one to ``margin[l]``."""
    for l in range(theta.shape[0]):
        y = theta[l].double()
        xi, _ = mq_decode(codes_all[lo + l], y, B, bits)
        acc = torch.zeros_like(y)
        hits = 0
        for j in nbrs[l]:
            xj, off = mq_decode(codes_all[j], y, B, bits)
            acc = acc + float(w_rows[l, j]) * (xj - xi)
            hits += int(mq_margin_hits(off, bits).sum())
        theta[l] = (y + acc).to(theta.dtype)
        margin[l] += hits


def mq_step_(theta: torch.Tensor, psi: Optional[torch.Tensor], grad: torch.Tensor, alpha: float, first: bool, B: float,
             bits: int, key, k: int, nodes, live: torch.Tensor) -> torch.Tensor:
    """The step of round ``k`` on the mixed rows, DSGD's (``psi`` None) or Exact Diffusion's (``ed_step_``, with
    ``psi <- theta`` first in round 0); returns the code rows published for round ``k + 1``."""
    if psi is None:
        dsgd_step_(theta, grad, alpha)
    else:
        if first:
            psi.copy_(theta)
        ed_step_(theta, psi, grad, alpha)
    return mq_encode(theta, B, bits, key, k + 1, nodes, live)


def mq_edge_gap(theta_all: torch.Tensor, edges, theta_bound: float) -> float:
    """``max over edges {i, j} of |theta_j - theta_i|_inf / theta_bound`` (0 without an edge): above 1 the run has left
    the decode guarantee."""
    gap = 0.0
    for i, j in edges:
        if i != j:
            gap = max(gap, float((theta_all[j].double() - theta_all[i].double()).abs().max()))
    return gap / float(theta_bound)


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
