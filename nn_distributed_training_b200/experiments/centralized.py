"""Centralized baselines: one model trained on the union of every node's data
(reference: centralized/*.ipynb — the 0.985 MNIST accuracy and the 2.34 online-density validation
loss drawn as reference lines in its figures, BASELINE.md).

    python -m nn_distributed_training_b200.experiments.centralized mnist <config.yaml> [--backend torch|fused]
    python -m nn_distributed_training_b200.experiments.centralized density <config.yaml> [--backend torch|fused]

``--backend fused`` trains on the sm_90a kernels (ops/local_train.py); its batches come from the in-kernel sampler
instead of ``torch.randperm``.
"""
from __future__ import annotations

import argparse

import numpy as np
import torch

from . import common
from . import density_common as dc
from ..data.mnist import load_mnist
from ..data.shards import Shard
from ..models import FourierNet, MNISTConvNet
from ..ops import local_train
from ..utils.config import load_experiment


def train_centralized(model, loss, train: Shard, val: Shard, device, epochs=6, lr=0.005, batch=100, val_batch=128,
                      squeeze=False, verbose=True, backend="torch", seed=0):
    """Adam on the union shard, evaluated after every epoch; ``backend``: torch (autograd) | fused (sm_90a kernels,
    ``ValueError`` when they cannot run this model / device)."""
    if backend not in local_train.BACKENDS:
        raise ValueError(f"backend must be one of {'|'.join(local_train.BACKENDS)} (got {backend!r})")
    if backend == "fused":
        return local_train.centralized(model, loss, train, val, device, epochs, lr, batch, val_batch, squeeze,
                                       verbose=verbose, seed=seed)
    model = model.to(device)
    dtype = next(model.parameters()).dtype
    opt = torch.optim.Adam(model.parameters(), lr=lr)
    tr, va = train.to(device), val.to(device)
    hist = []
    for ep in range(epochs):
        perm = torch.randperm(len(tr), device=device)
        for a in range(0, len(tr), batch):
            idx = perm[a: a + batch]
            out = model(tr.inputs(idx, dtype))
            y = tr.targets(idx)
            l = loss(torch.squeeze(out), y.to(dtype)) if squeeze else loss(out, y)
            opt.zero_grad(); l.backward(); opt.step()
        with torch.no_grad():
            vloss, correct = 0.0, 0
            for a in range(0, len(va), val_batch):
                idx = torch.arange(a, min(len(va), a + val_batch), device=device)
                out = model(va.inputs(idx, dtype))
                y = va.targets(idx)
                vloss += (loss(torch.squeeze(out), y.to(dtype)) if squeeze else loss(out, y)).item()
                if not squeeze:
                    correct += out.argmax(1).eq(y).sum().item()
        rec = {"epoch": ep, "validation_loss": vloss, "top1_accuracy": correct / len(va) if not squeeze else None}
        hist.append(rec)
        if verbose:
            print(rec)
    return hist


def centralized_mnist(yaml_pth, backend="torch"):
    conf = load_experiment(yaml_pth, "mnist")["experiment"]
    ctx = common.make_context(conf)
    train, _ = load_mnist(conf["data_dir"], True)
    val, _ = load_mnist(conf["data_dir"], False)
    m = conf["model"]
    solo = conf["individual_training"]
    return train_centralized(MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"]), common.make_loss(conf["loss"]),
                             train, val, ctx.device, epochs=solo["epochs"], lr=solo["lr"], batch=solo["train_batch_size"],
                             val_batch=solo["val_batch_size"], backend=backend, seed=int(conf.get("seed", 0)))


def centralized_density(yaml_pth, online=True, backend="torch"):
    from ..floorplans.lidar import RandomPoseLidarDataset, TrajectoryLidarDataset
    conf = load_experiment(yaml_pth, "online_density" if online else "density")["experiment"]
    ctx = common.make_context(conf)
    data_conf = conf["data"]
    data_dir = dc.resolve_data_dir(data_conf, ctx)
    lidar = dc.make_lidar(data_conf, data_dir, device=ctx.device)
    paths = dc.waypoint_files(data_dir, data_conf["waypoint_subdir"])
    sets = [TrajectoryLidarDataset(lidar, np.load(p), data_conf["spline_res"], round_density=data_conf["round_density"]) for p in paths]
    train = Shard(torch.cat([s.shard.x for s in sets]), torch.cat([s.shard.y for s in sets]))
    val = RandomPoseLidarDataset(lidar, data_conf["num_validation_scans"], round_density=data_conf["round_density"]).shard
    solo = conf["individual_training"]
    model = FourierNet(conf["model"]["shape"], scale=conf["model"]["scale"])
    return train_centralized(model, common.make_loss(conf["loss"]), train, val, ctx.device, epochs=solo["epochs"], lr=solo["lr"],
                             batch=solo["train_batch_size"], val_batch=solo["val_batch_size"], squeeze=True,
                             backend=backend, seed=int(conf.get("seed", 0)))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("kind", choices=("mnist", "density", "offline_density"))
    ap.add_argument("config")
    ap.add_argument("--backend", choices=local_train.BACKENDS, default="torch")
    args = ap.parse_args(argv)
    if args.kind == "mnist":
        return centralized_mnist(args.config, backend=args.backend)
    return centralized_density(args.config, online=(args.kind != "offline_density"), backend=args.backend)


if __name__ == "__main__":
    main()
