"""DSGD, DSGT and RelaySum on the PAPER MNIST setup with heterogeneous data, on a 10-node path and a 10-node binary
tree: device time per round, bytes per round and final accuracy.

    python scripts/bench_relaysum.py [--graphs path,binary_tree] [--dtypes fp64,fp32] [--rounds 400] [--warmup 40]
                                     [--repeats 3] [--accuracy-rounds 2000] [--accuracy-dtypes fp32]
                                     [--sweep 0.001,0.005,0.02] [--sweep-rounds 2000]
                                     [--data-source auto|mnist|synthetic|synthetic_hard] [--out FILE.json]

The problems are those of ``experiments/dist_mnist_relaysum.yaml``: 10 nodes, the heterogeneous class split,
MNISTConvNet(3, 5, 64), batch 64, on the fused sm_90a kernels, on each graph of ``--graphs``.  The default data source is ``synthetic_hard``, the
synthetic set on which DSGD's bias under heterogeneous data shows; ``auto`` takes MNIST from ``--data-dir`` if it is
there and the separable synthetic images otherwise.  The source is printed.
  * speed: for each graph and dtype the three runs alternate ``--repeats`` times; each builds its problem, runs
    ``--warmup`` rounds, captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA
    events (ms per round, the median over repeats);
  * bytes: the engine's ``bytes_per_round()`` of each run (one published row, and the rows a rank pulls per round);
  * ``--sweep``: the three runs at each step size (``alpha0`` of DSGD and RelaySum, ``alpha`` of DSGT) for
    ``--sweep-rounds`` rounds (fp32), mean top-1 at the end;
  * accuracy: one run of ``--accuracy-rounds`` rounds per run, graph and dtype, the runs one after the other; the mean over
    nodes of the top-1 accuracy at the last evaluation (the start of the final round, as the runner reports it).
The card's name and power limit are printed in the same run.  Prints one JSON line (and writes it to ``--out``).
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.experiments.dist_mnist_ex import split_hetero  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_relaysum.yaml")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--graphs", default="path,binary_tree")
    ap.add_argument("--dtypes", default="fp64,fp32")
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--accuracy-dtypes", default="fp32")
    ap.add_argument("--sweep", default="")
    ap.add_argument("--sweep-rounds", type=int, default=2000)
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="synthetic_hard", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_relaysum.py measures the fused kernels and needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    N = int(exp["graph"]["num_nodes"])
    train, src = load_mnist(args.data_dir, train=True, source=args.data_source)
    val, _ = load_mnist(args.data_dir, train=False, source=args.data_source)
    shards = split_hetero(train, N)
    print(f"MNIST source: {src} ({len(train)} train / {len(val)} val), {N} nodes", flush=True)
    problems = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}
    algs = list(problems)

    def build(graph, alg, dtype, rounds, eval_every, alpha=None):
        pc = copy.deepcopy(problems[alg])
        pc["optimizer_config"]["outer_iterations"] = rounds
        if alpha is not None:
            pc["optimizer_config"]["alpha" if alg == "dsgt" else "alpha0"] = alpha
        pc["metrics_config"]["evaluate_frequency"] = eval_every
        torch.manual_seed(0)
        m = exp["model"]
        model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
        pr = DistMNISTProblem(graph, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
        opt = build_optimizer(pr, dev, pc["optimizer_config"])
        assert opt._use_engine(), f"{alg} does not run on the fused consensus kernels"
        return pr, opt

    def top1(pr):
        return round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1], dtype=torch.float64).mean()), 4)

    record = {"card": gpu, "data_source": src, "nodes": N, "speed_ms_per_round": {}, "bytes_per_round": {},
              "accuracy": {}, "sweep": {}, "rounds": args.rounds, "warmup": args.warmup, "repeats": args.repeats}
    for gname in args.graphs.split(","):
        _, graph = graph_generation.generate_from_conf({"type": gname, "num_nodes": N})
        for dname in args.dtypes.split(","):
            times = {a: [] for a in algs}
            for _ in range(args.repeats):
                for alg in algs:
                    pr, opt = build(graph, alg, DTYPES[dname], args.warmup + args.rounds, 10 ** 9)
                    opt.run_rounds(args.warmup)
                    opt.prepare_rounds(args.rounds)
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    t0.record()
                    opt.run_rounds(args.rounds)
                    t1.record()
                    torch.cuda.synchronize()
                    opt._program.eng.check()
                    times[alg].append(round(t0.elapsed_time(t1) / args.rounds, 4))
                    record["bytes_per_round"].setdefault(gname, {}).setdefault(dname, {})[alg] = \
                        opt._program.eng.bytes_per_round()
                    del pr, opt
            med = {a: statistics.median(v) for a, v in times.items()}
            record["speed_ms_per_round"].setdefault(gname, {})[dname] = {"median": med, "all": times}
            print(f"{gname} {dname}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in algs) + f"   (all {times})",
                  flush=True)
            print(f"{gname} {dname}: bytes/round {record['bytes_per_round'][gname][dname]}", flush=True)

        for alpha in [float(x) for x in args.sweep.split(",") if x]:
            for alg in algs:
                pr, opt = build(graph, alg, torch.float32, args.sweep_rounds, args.sweep_rounds, alpha=alpha)
                opt.train()
                record["sweep"].setdefault(gname, {}).setdefault(alg, {})[alpha] = top1(pr)
                print(f"sweep {gname} fp32 {alg} alpha {alpha}: mean top-1 after {args.sweep_rounds} rounds "
                      f"{top1(pr):.4f}", flush=True)
                del pr, opt

        for dname in (args.accuracy_dtypes.split(",") if args.accuracy_rounds > 0 else []):
            acc = {}
            for alg in algs:
                pr, opt = build(graph, alg, DTYPES[dname], args.accuracy_rounds, args.accuracy_rounds)
                opt.train()
                acc[alg] = top1(pr)
                del pr, opt
            record["accuracy"].setdefault(gname, {})[dname] = acc
            print(f"{gname} {dname}: mean top-1 after {args.accuracy_rounds} rounds ({src}): "
                  + "  ".join(f"{a} {acc[a]:.4f}" for a in algs), flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
