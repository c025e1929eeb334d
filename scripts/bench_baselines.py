"""Wall time of the no-communication baselines on the torch (autograd) and fused (sm_90a kernels) backends.

    python scripts/bench_baselines.py [--dtypes fp64,fp32] [--repeats 3] [--out FILE.json]

In one process, for each dtype, the two backends alternate ``--repeats`` times on:
  * ``solo_density``: the solo baseline of ``experiments/dist_online_dense_PAPER.yaml`` (7 nodes, 1 epoch of each
    node's trajectory shard at batch 10,000, Adam lr 1e-3) on the shipped floor plan ``floorplans/32_data``;
  * ``central_mnist``: centralized MNISTConvNet(3, 5, 64) on 60,000 synthetic MNIST images, 6 epochs at batch 100,
    Adam lr 5e-3, evaluated on 10,000 after every epoch;
  * ``central_density``: centralized online density, one model on the union of the 7 trajectory shards, the PAPER's
    individual_training settings.
Each timing is host wall time from a device synchronise to a device synchronise around the whole call: training,
evaluation and, for the fused backend, building the problem and capturing its graphs.  Data generation is outside.
The card's name and power limit are printed with the numbers.  Prints one JSON line (and writes it to ``--out``).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nn_distributed_training_b200.data.mnist import synthetic_mnist  # noqa: E402
from nn_distributed_training_b200.data.shards import Shard  # noqa: E402
from nn_distributed_training_b200.experiments import centralized, common  # noqa: E402
from nn_distributed_training_b200.experiments import density_common as dc  # noqa: E402
from nn_distributed_training_b200.floorplans.lidar import OnlineTrajectoryLidarDataset, RandomPoseLidarDataset  # noqa: E402
from nn_distributed_training_b200.models import FourierNet, MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.parallel.context import DistContext  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def density_data(dev):
    with open(os.path.join(ROOT, "experiments", "dist_online_dense_PAPER.yaml")) as f:
        exp = yaml.safe_load(f)["experiment"]
    data_conf = dict(exp["data"], data_dir=os.path.join(ROOT, "floorplans", "32_data"))
    ctx = DistContext.single(dev)
    data_dir = dc.resolve_data_dir(data_conf, ctx)
    lidar = dc.make_lidar(data_conf, data_dir, device=dev)
    paths = dc.waypoint_files(data_dir, data_conf["waypoint_subdir"])
    train = [OnlineTrajectoryLidarDataset(lidar, np.load(p), data_conf["spline_res"], data_conf["num_scans_in_window"],
                                          round_density=data_conf["round_density"], seed=int(exp["seed"]), node=i)
             for i, p in enumerate(paths)]
    val = RandomPoseLidarDataset(lidar, data_conf["num_validation_scans"], round_density=data_conf["round_density"])
    return exp, train, val


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--dtypes", default="fp64,fp32")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--workloads", default="solo_density,central_mnist,central_density")
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_baselines.py measures the GPU baselines and needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = card()
    print(f"card: {gpu}", flush=True)
    workloads = args.workloads.split(",")

    exp, dtrain, dval = density_data(dev) if {"solo_density", "central_density"} & set(workloads) else (None, None, None)
    if exp is not None:
        solo = dict(exp["individual_training"], verbose=False)
        loss_d = common.make_loss(exp["loss"])
        union = Shard(torch.cat([s.shard.x for s in dtrain]), torch.cat([s.shard.y for s in dtrain]))
        print(f"density: {len(dtrain)} nodes, shards {[len(s.shard) for s in dtrain]}, union {len(union)}", flush=True)
    mtrain, mval = synthetic_mnist(60000, seed=0), synthetic_mnist(10000, seed=1)

    def run(work, dtype, backend):
        torch.manual_seed(0)
        if work == "solo_density":
            model = FourierNet(exp["model"]["shape"], scale=exp["model"]["scale"], dtype=dtype)
            return dc.solo_results(model, loss_d, dtrain, dval, dev, dict(solo, backend=backend), seed=0)
        if work == "central_mnist":
            return centralized.train_centralized(MNISTConvNet(3, 5, 64, dtype=dtype), torch.nn.NLLLoss(), mtrain, mval,
                                                 dev, epochs=6, lr=0.005, batch=100, val_batch=100, verbose=False,
                                                 backend=backend)
        model = FourierNet(exp["model"]["shape"], scale=exp["model"]["scale"], dtype=dtype)
        return centralized.train_centralized(model, loss_d, union, dval.shard, dev, epochs=solo["epochs"], lr=solo["lr"],
                                             batch=solo["train_batch_size"], val_batch=solo["val_batch_size"],
                                             squeeze=True, verbose=False, backend=backend)

    def summary(work, out):
        if work == "solo_density":
            return [round(float(out[g]["validation_loss"]), 4) for g in sorted(out)]
        return [round(float(h["validation_loss"]), 4) for h in out][-1:] + (
            [h["top1_accuracy"] for h in out][-1:] if work == "central_mnist" else [])

    record = {"card": gpu, "repeats": args.repeats, "results": {}}
    for dname in args.dtypes.split(","):
        dtype = DTYPES[dname]
        for work in workloads:
            times = {"torch": [], "fused": []}
            last = {}
            for _ in range(args.repeats):
                for backend in ("torch", "fused"):
                    t, out = timed(lambda: run(work, dtype, backend))
                    times[backend].append(round(t, 4))
                    last[backend] = summary(work, out)
            med = {b: statistics.median(v) for b, v in times.items()}
            rec = {"torch_s": med["torch"], "fused_s": med["fused"], "speedup": round(med["torch"] / med["fused"], 2),
                   "times": times, "val": last}
            record["results"][f"{work}/{dname}"] = rec
            print(f"{work:16s} {dname}: torch {med['torch']:.3f} s  fused {med['fused']:.3f} s  "
                  f"x{rec['speedup']}  (all {times})  val {last}", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
