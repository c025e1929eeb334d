"""ClippedGossip and BRIDGE against Byzantine nodes on the setup of ``experiments/dist_mnist_byzantine.yaml`` (10-node
complete graph through the neighbor pointer table, heterogeneous class split, MNISTConvNet(3, 5, 64), batch 64, nodes 0
and 1 attacking, delta 0.2; the BRIDGE arms of ``experiments/dist_mnist_bridge.yaml``, trimmed mean with b 2 and
median, on the same setup), on the fused sm_90a kernels.  Device time per round, bytes read per round, and the honest
nodes' accuracy.

    python scripts/bench_byzantine.py [--dtypes fp64,fp32] [--rounds 400] [--warmup 40] [--repeats 3]
                                      [--accuracy-rounds 2000] [--accuracy-dtype fp32]
                                      [--data-source auto|mnist|synthetic|synthetic_hard] [--out FILE.json]

  * speed: for each dtype the arms DSGD, ``clip: none``, ``clip: adaptive``, BRIDGE ``trimmed_mean`` (``bridge_tm``) and
    BRIDGE ``median`` (no attacker) alternate ``--repeats``
    times; each builds its problem, runs ``--warmup`` rounds, captures the CUDA graphs of the next ``--rounds`` rounds
    and times their replay with CUDA events (ms per round, the median over repeats);
  * bytes: what this process's nodes read from their neighbors per round, from the engine (computed, not measured);
  * accuracy: one run of ``--accuracy-rounds`` rounds per arm (DSGD without attack; ``clip: none``, ``adaptive`` and
    the two BRIDGE screens under ``sign_flip`` and ``alie``), arms alternated in this process; mean and worst top-1
    over the honest nodes at the last evaluation.
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
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_byzantine.yaml")
BRIDGE_YAML = os.path.join(ROOT, "experiments", "dist_mnist_bridge.yaml")
SPEED = ["dsgd", "cg_none", "cg_adaptive", "bridge_tm", "bridge_median"]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--dtypes", default="fp64,fp32")
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--accuracy-dtype", default="fp32")
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="auto", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_byzantine.py measures the fused kernels and needs a CUDA device")
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
    bridge = load_experiment(BRIDGE_YAML, "mnist")       # the same experiment block; its BRIDGE arms only
    problems.update({pc["problem_name"]: pc for pc in bridge["problem_configs"].values()
                     if pc["optimizer_config"]["alg_name"] == "bridge"})
    for name in SPEED[1:]:                       # the speed arms: no attacker
        pc = problems[name] = copy.deepcopy(problems[f"{name}_sign_flip"])
        pc["problem_name"] = name
        del pc["optimizer_config"]["byzantine"]

    def build(name, dtype, rounds, eval_every):
        pc = copy.deepcopy(problems[name])
        pc["optimizer_config"]["outer_iterations"] = rounds
        pc["metrics_config"]["evaluate_frequency"] = eval_every
        torch.manual_seed(0)
        m = exp["model"]
        model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
        pr = DistMNISTProblem(graph, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
        opt = build_optimizer(pr, dev, pc["optimizer_config"])
        assert opt._use_engine(), f"{name} does not run on the fused consensus kernels"
        return pr, opt

    record = {"card": gpu, "data_source": src, "nodes": N, "graph": exp["graph"]["type"], "speed_ms_per_round": {},
              "bytes_computed": {}, "accuracy": {}, "rounds": args.rounds, "warmup": args.warmup,
              "repeats": args.repeats, "multi_gpu": "not measured"}
    for dname in [d for d in args.dtypes.split(",") if d]:
        times = {a: [] for a in SPEED}
        for _ in range(args.repeats):
            for name in SPEED:
                pr, opt = build(name, DTYPES[dname], args.warmup + args.rounds, 10 ** 9)
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
                record["bytes_computed"].setdefault(dname, {})[name] = opt._program.eng.bytes_per_round()["pulled"]
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        record["speed_ms_per_round"][dname] = {"median": med, "all": times}
        print(f"{dname}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in SPEED) + f"   (all {times})", flush=True)
        print(f"{dname}: bytes read per round (computed) "
              + "  ".join(f"{a} {b}" for a, b in record["bytes_computed"][dname].items()), flush=True)

    if args.accuracy_rounds > 0:
        for name in problems:
            if name in SPEED[1:]:
                continue
            pr, opt = build(name, DTYPES[args.accuracy_dtype], args.accuracy_rounds, args.accuracy_rounds)
            opt.train()
            acc = torch.as_tensor(pr.metrics["top1_accuracy"][-1], dtype=torch.float64).reshape(-1)
            honest = [i for i in range(N) if i not in set(getattr(opt, "byzantine", []))]
            a = acc[honest]
            record["accuracy"][name] = {"honest_mean": round(float(a.mean()), 4), "honest_worst": round(float(a.min()), 4)}
            print(f"{args.accuracy_dtype} {name}: honest top-1 after {args.accuracy_rounds} rounds ({src}) "
                  f"mean {float(a.mean()):.4f} worst {float(a.min()):.4f}", flush=True)
            del pr, opt
    print("multi-GPU: not measured", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
