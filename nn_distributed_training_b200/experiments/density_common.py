"""Shared helpers of the lidar density runners."""
from __future__ import annotations

import copy
import glob
import os

import numpy as np
import torch

from . import common
from ..floorplans import synthetic
from ..floorplans.lidar import ClippedLidar2D, Lidar2D


def resolve_data_dir(data_conf, ctx) -> str:
    """Use ``data_dir`` when it holds ``floor_img.png``; otherwise (or when
    ``data_dir: synthetic``) generate a procedural floor plan + waypoint sets in the
    reference's layout under ``synthetic_dir`` (there are no data files in this repo)."""
    d = data_conf["data_dir"]
    if d != "synthetic" and os.path.exists(os.path.join(d, "floor_img.png")):
        return d
    out = data_conf.get("synthetic_dir", os.path.join(os.path.dirname(__file__), "..", "floorplans", "_synthetic_data"))
    out = os.path.abspath(out)
    sub = data_conf.get("waypoint_subdir", "tight_paths")
    if ctx.is_main and not os.path.exists(os.path.join(out, sub)):
        synthetic.write_dataset(out, n_paths=int(data_conf.get("synthetic_paths", 8)), subdir=sub,
                                seed=int(data_conf.get("synthetic_seed", 0)))
    ctx.barrier()
    if ctx.is_main:
        print(f"floor plan: synthetic ({out})")
    return out


def make_lidar(data_conf, data_dir, clipped=False, device=None):
    """``device``: a CUDA device makes ``Lidar2D`` generate its scans with ops/csrc/lidar.cu
    (``data_conf['lidar_backend']``: auto | cuda | numpy)."""
    lidar = _make_lidar(data_conf, data_dir, clipped)
    backend = str(data_conf.get("lidar_backend", "auto"))
    if backend != "numpy" and not clipped and device is not None and torch.device(device).type == "cuda":
        from ..ops import fused_available
        if fused_available() or backend == "cuda":
            lidar.scan_device = torch.device(device)
    return lidar


def _make_lidar(data_conf, data_dir, clipped=False):
    img_path = os.path.join(data_dir, "floor_img.png")
    if clipped:
        return ClippedLidar2D(img_path, data_conf["num_beams"], data_conf["beam_length"], data_conf["beam_samps"],
                              border_width=data_conf["border_width"])
    return Lidar2D(img_path, data_conf["num_beams"], data_conf["beam_length"], data_conf["beam_samps"],
                   data_conf["samp_distribution_factor"], data_conf["collision_samps"], data_conf["fine_samps"],
                   border_width=data_conf["border_width"])


def waypoint_files(data_dir, subdir):
    return sorted(glob.glob(os.path.join(data_dir, subdir, "*.npy")))


def mesh_inputs(val_set, device, dtype):
    X, Y = np.meshgrid(val_set.lidar.xs, val_set.lidar.ys)
    mesh = np.hstack((X[::8, ::8].reshape(-1, 1), Y[::8, ::8].reshape(-1, 1)))
    return torch.as_tensor(mesh, dtype=dtype, device=device)


def solo_results(base_model, loss, train_sets, val_set, device, conf, seed=0):
    """``{node: train_solo result}`` of every node, on the backend ``conf['backend']`` names (torch | fused)."""
    if conf["backend"] == "fused":
        from ..ops import local_train
        return local_train.solo_density(base_model, loss, train_sets, val_set, device, conf, seed=seed)
    return {i: train_solo(copy.deepcopy(base_model), loss, s, val_set, device, conf) for i, s in enumerate(train_sets)}


def train_solo(model, loss, train_set, val_set, device, conf):
    """Single-node baseline (reference: experiments/dist_online_dense_ex.py:30-90)."""
    model = model.to(device)
    dtype = next(model.parameters()).dtype
    opt = common.make_solo_optimizer(model, conf)
    tr = train_set.shard.to(device)
    va = val_set.shard.to(device)
    n, bs = len(tr), int(conf["train_batch_size"])
    for _ in range(int(conf["epochs"])):
        perm = torch.randperm(n, device=device)
        for a in range(0, n, bs):
            idx = perm[a: a + bs]
            opt.zero_grad()
            l = loss(torch.squeeze(model(tr.x[idx].to(dtype))), tr.y[idx].to(dtype))
            l.backward()
            opt.step()
    with torch.no_grad():
        vloss = torch.zeros((), device=device, dtype=dtype)
        vb = int(conf["val_batch_size"])
        for a in range(0, len(va), vb):
            vloss += loss(torch.squeeze(model(va.x[a: a + vb].to(dtype))), va.y[a: a + vb].to(dtype))
        mesh = mesh_inputs(val_set, device, dtype)
        dense = model(mesh)
    # CPU tensors: solo_results.pt must load on a machine without a GPU (the notebooks / visualization tools)
    return {"validation_loss": vloss.cpu(), "mesh_grid_density": dense.cpu(), "mesh_grid": mesh.cpu()}
