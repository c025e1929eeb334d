"""Local steps on the PAPER MNIST setup: DiNNO (2 primal steps), DSGD, DSGT, and local DSGD and K-GT at K = 1, 2 and
4 local steps per round.  Device time per round and per gradient step, bytes pulled per round and per gradient step,
and final accuracy.

    python scripts/bench_local_steps.py [--dtypes fp64,fp32] [--rounds 400] [--warmup 40] [--repeats 3]
                                        [--accuracy-rounds 2000] [--accuracy-dtypes fp32]
                                        [--sweep 0.002,0.005,0.01,0.02] [--sweep-rounds 500]
                                        [--data-source auto|mnist|synthetic|synthetic_hard] [--out FILE.json]

The problems are those of ``experiments/dist_mnist_local_steps.yaml`` (a 10-node cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), batch 64, on the fused sm_90a kernels), with DSGD taken from ``dist_mnist_PAPER.yaml`` and the
K = 1 and K = 4 arms added to local DSGD and K-GT.  Their alpha is DSGT's 0.005 and is not tuned.
  * speed: for each dtype the nine arms alternate ``--repeats`` times; each builds its problem, runs ``--warmup``
    rounds, captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA events (ms per
    round, the median over repeats; per gradient step: divided by the draws per round);
  * bytes: everything this process's nodes pull per round, from the engine (computed, not measured), and per gradient
    step;
  * ``--sweep``: the local-DSGD and K-GT arms at K = 2 and 4, ``--sweep-rounds`` rounds at each alpha (fp32), mean
    top-1 at the end;
  * accuracy: one run of ``--accuracy-rounds`` rounds per arm and dtype; the mean over nodes of the top-1 accuracy at
    the last evaluation.
The card's name and power limit are printed in the same run.  Prints one JSON line (and writes it to ``--out``).
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_algorithms import card  # noqa: E402
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.experiments.dist_mnist_ex import split_hetero  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.ops.round_program import draws_per_round  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_local_steps.yaml")
PAPER = os.path.join(ROOT, "experiments", "dist_mnist_PAPER.yaml")
NAMES = ["dinno", "dsgd", "dsgt", "local_dsgd_k1", "local_dsgd_k2", "local_dsgd_k4", "kgt_k1", "kgt_k2", "kgt_k4"]
SWEPT = ["local_dsgd_k2", "local_dsgd_k4", "kgt_k2", "kgt_k4"]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--dtypes", default="fp64,fp32")
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--accuracy-dtypes", default="fp32")
    ap.add_argument("--sweep", default="")
    ap.add_argument("--sweep-rounds", type=int, default=500)
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="auto", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_local_steps.py measures the fused kernels and needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    N, graph = graph_generation.generate_from_conf(exp["graph"])
    train, src = load_mnist(args.data_dir, train=True, source=args.data_source)
    val, _ = load_mnist(args.data_dir, train=False, source=args.data_source)
    shards = split_hetero(train, N)
    print(f"MNIST source: {src} ({len(train)} train / {len(val)} val), {N} nodes, {exp['graph']['type']}", flush=True)
    problems = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}
    problems["dsgd"] = next(pc for pc in load_experiment(PAPER, "mnist")["problem_configs"].values()
                            if pc["optimizer_config"]["alg_name"] == "dsgd")
    for corr, base in ((False, "local_dsgd"), (True, "kgt")):
        for K in (1, 4):
            pc = problems[f"{base}_k{K}"] = copy.deepcopy(problems[f"{base}_k2"])
            pc["problem_name"] = f"{base}_k{K}"
            pc["optimizer_config"]["local_steps"] = K

    def build(name, dtype, rounds, eval_every, alpha=None):
        pc = copy.deepcopy(problems[name])
        pc["optimizer_config"]["outer_iterations"] = rounds
        if alpha is not None:
            pc["optimizer_config"]["alpha"] = alpha
        pc["metrics_config"]["evaluate_frequency"] = eval_every
        torch.manual_seed(0)
        m = exp["model"]
        model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
        pr = DistMNISTProblem(graph, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
        opt = build_optimizer(pr, dev, pc["optimizer_config"])
        assert opt._use_engine(), f"{name} does not run on the fused consensus kernels"
        return pr, opt

    def top1(pr):
        return round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1], dtype=torch.float64).mean()), 4)

    record = {"card": gpu, "data_source": src, "nodes": N, "graph": exp["graph"]["type"], "speed_ms_per_round": {},
              "speed_ms_per_step": {}, "bytes_computed": {}, "accuracy": {}, "sweep": {}, "rounds": args.rounds,
              "warmup": args.warmup, "repeats": args.repeats, "multi_gpu": "not measured"}
    steps = {}
    for dname in [d for d in args.dtypes.split(",") if d]:
        times = {a: [] for a in NAMES}
        for _ in range(args.repeats):
            for name in NAMES:
                pr, opt = build(name, DTYPES[dname], args.warmup + args.rounds, 10 ** 9)
                steps[name] = draws_per_round(opt)
                opt.run_rounds(args.warmup)
                opt.prepare_rounds(args.rounds)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0.record()
                opt.run_rounds(args.rounds)
                t1.record()
                torch.cuda.synchronize()
                opt._program.eng.check()
                times[name].append(round(t0.elapsed_time(t1) / args.rounds, 4))
                pulled = opt._program.eng.bytes_per_round()["pulled"]
                record["bytes_computed"].setdefault(dname, {})[name] = {
                    "pulled_per_round": pulled, "pulled_per_step": pulled / steps[name], "steps_per_round": steps[name]}
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        record["speed_ms_per_round"][dname] = {"median": med, "all": times}
        record["speed_ms_per_step"][dname] = {a: round(med[a] / steps[a], 5) for a in NAMES}
        print(f"{dname}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in NAMES) + f"   (all {times})", flush=True)
        print(f"{dname}: ms/gradient step " + "  ".join(f"{a} {v:.4f}" for a, v in record["speed_ms_per_step"][dname].items()),
              flush=True)
        print(f"{dname}: bytes pulled per round / per gradient step (computed) "
              + "  ".join(f"{a} {b['pulled_per_round']}/{b['pulled_per_step']:.0f}"
                          for a, b in record["bytes_computed"][dname].items()), flush=True)

    for alpha in [float(x) for x in args.sweep.split(",") if x]:
        for name in SWEPT:
            pr, opt = build(name, torch.float32, args.sweep_rounds, args.sweep_rounds, alpha=alpha)
            opt.train()
            record["sweep"].setdefault(name, {})[alpha] = top1(pr)
            print(f"sweep fp32 {name} alpha {alpha}: mean top-1 after {args.sweep_rounds} rounds {top1(pr):.4f}", flush=True)
            del pr, opt

    for dname in (args.accuracy_dtypes.split(",") if args.accuracy_rounds > 0 else []):
        acc = {}
        for name in NAMES:
            pr, opt = build(name, DTYPES[dname], args.accuracy_rounds, args.accuracy_rounds)
            opt.train()
            acc[name] = top1(pr)
            del pr, opt
        record["accuracy"][dname] = acc
        print(f"{dname}: mean top-1 after {args.accuracy_rounds} rounds ({src}): "
              + "  ".join(f"{a} {acc[a]:.4f}" for a in NAMES), flush=True)
    print("multi-GPU: not measured (one GPU)" if torch.cuda.device_count() < 2 else
          "multi-GPU: not measured by this script", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
