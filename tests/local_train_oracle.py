"""Oracles of the fused local-training path (``ops/local_train.py``).

* ``local_step``: float64 NumPy oracle of one ``local_step`` launch (csrc/consensus.cu: local_step_kernel) with the
  first-order error bound of ``tests/consensus_oracle.py``: the node's S partials summed, one SGD / Adam / AdamW step
  at t = calls + 1, calls advanced; a node at its budget is unchanged (bound 0: bitwise).
* ``HostTwinTrainer``: torch.optim on the batches the in-kernel sampler draws, read from its host twin
  ``data.sampler.BatchSchedule`` — the autograd run the fused solo / centralized baselines are compared with.
* ``feistel_randperm``: a ``torch.randperm`` stand-in that hands the torch loops the same epoch permutations.
"""
from __future__ import annotations

import numpy as np
import torch

import consensus_oracle as co
from nn_distributed_training_b200.data.sampler import BatchSchedule, feistel_permute, mix_key
from nn_distributed_training_b200.experiments import common


def local_step(st, *, opt, lr, u, dtype):
    """One launch on ``st`` (theta / m / v ``[L, n]``, grad_part ``[L, S, n]``, calls / budget ``[L]``)."""
    L = st["theta"].shape[0]
    out = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}
    err = {k: np.zeros_like(st[k]) for k in ("theta", "m", "v") if st.get(k) is not None}
    gl, e_gl = co.sum_partials(st["grad_part"], u)
    b1, b2, eps, wd = co.adam_constants(dtype)
    lr = float(np.dtype(dtype).type(lr))
    for i in range(L):
        call = int(st["calls"][i])
        if call >= int(st["budget"][i]):
            continue
        th, g, e_g = st["theta"][i], gl[i], e_gl[i]
        if opt == "sgd":
            new = th - lr * g
            e_new = u * (np.abs(th) + 2.0 * lr * np.abs(g)) + lr * e_g
        else:
            m0, v0 = st["m"][i], st["v"][i]
            m = b1 * m0 + (1.0 - b1) * g
            e_m = u * (b1 * np.abs(m0) + (1.0 - b1) * np.abs(g) + np.abs(m)) + (1.0 - b1) * e_g
            v = b2 * v0 + (1.0 - b2) * g * g
            e_v = u * (b2 * v0 + 2.0 * (1.0 - b2) * g * g + v) + (1.0 - b2) * 2.0 * np.abs(g) * e_g
            step_v, e_step = co.adam_step(m, v, e_m, e_v, lr=lr, t=call + 1, u=u, b1=b1, b2=b2, eps=eps)
            base, e_base = th, np.zeros_like(th)
            if opt == "adamw":
                base = th * (1.0 - lr * wd)
                e_base = 2.0 * u * np.abs(th)
            new = base - step_v
            e_new = e_base + e_step + u * (np.abs(base) + np.abs(step_v))
            out["m"][i], err["m"][i] = m, e_m
            out["v"][i], err["v"][i] = v, e_v
        out["theta"][i], err["theta"][i] = new, e_new
        out["calls"][i] = call + 1
    return out, err


class HostTwinTrainer:
    """``model`` trained alone with the solo optimizer on node ``node``'s sampler stream (call by call)."""

    def __init__(self, model, loss, shard, batch, optimizer, lr, seed, node, squeeze=False):
        self.model, self.loss, self.shard, self.squeeze = model, loss, shard, squeeze
        self.opt = common.make_solo_optimizer(model, {"optimizer": optimizer, "lr": lr})
        self.sched = BatchSchedule(len(shard), int(batch))
        self.seed, self.node, self.call = int(seed), int(node), 0
        self.dtype = next(model.parameters()).dtype

    def run(self, steps):
        for _ in range(int(steps)):
            idx = self.sched.indices(self.call, self.seed, self.node, device=self.shard.x.device)
            out = self.model(self.shard.inputs(idx, self.dtype))
            y = self.shard.targets(idx)
            l = self.loss(torch.squeeze(out), y.to(self.dtype)) if self.squeeze else self.loss(out, y)
            self.opt.zero_grad()
            l.backward()
            self.opt.step()
            self.call += 1
        return self.model


def feistel_randperm(seed, node):
    """A ``torch.randperm(n, device=...)`` whose e-th call returns the sampler's epoch-e permutation of node ``node``."""
    state = {"epoch": 0}

    def randperm(n, device=None, **_):
        key = mix_key(int(seed), int(node), state["epoch"])
        state["epoch"] += 1
        return feistel_permute(torch.arange(n, dtype=torch.int64), n, key).to(device)

    return randperm


def flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])
