"""DSGT, CHOCO-SGD (int8 / sign) and BEER (compressor none / int8 / sign) on the PAPER MNIST setup: device time per
round, bytes published per row and pulled per round, and final accuracy.

    python scripts/bench_beer.py [--dtypes fp64,fp32] [--rounds 400] [--warmup 40] [--repeats 3]
                                 [--accuracy-rounds 2000] [--accuracy-dtypes fp32]
                                 [--sweep 0.1,0.3,0.5,0.8,1.0] [--sweep-rounds 500] [--gamma-from-sweep]
                                 [--data-source auto|mnist|synthetic|synthetic_hard] [--out FILE.json]
                                 [--topk 0.01,0.05] [--step-launches 2000]

The problems are those of ``experiments/dist_mnist_beer.yaml`` (a 10-node cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), batch 64, on the fused sm_90a kernels), with ``choco_sign`` added at CHOCO int8's gamma and
``beer_none`` at gamma 1 (DSGT's iterates with the own-tracker step and a zero tracker start).  BEER's alpha is DSGT's
and is not tuned.
  * speed: for each dtype the six configurations alternate ``--repeats`` times; each builds its problem, runs
    ``--warmup`` rounds, captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA
    events (ms per round, the median over repeats);
  * bytes: one published row per node (both channels) and everything this process's nodes pull per round, from the
    engine;
  * ``--sweep``: the compressed CHOCO and BEER runs of ``--sweep-rounds`` rounds at each gamma (fp32), mean top-1 at the
    end; with ``--gamma-from-sweep`` the accuracy runs take each of them at its best swept gamma (the first of a tie);
  * accuracy: one run of ``--accuracy-rounds`` rounds per configuration and dtype; the mean over nodes of the top-1
    accuracy at the last evaluation;
  * ``--topk``: ``choco_topk<ratio>`` and ``beer_topk<ratio>`` configurations per ratio (the int8 problems with
    compressor topk), measured, swept and run with the others; ``--step-launches``: the step kernels alone, int8
    against each top-k ratio, timed with CUDA events over that many back-to-back launches replayed from one CUDA graph
    (ms per launch, per dtype).
Without ``--topk`` the output is that of the six configurations above.
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
from bench_compression import step_kernel_times  # noqa: E402
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.experiments.dist_mnist_ex import split_hetero  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_beer.yaml")


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
    ap.add_argument("--gamma-from-sweep", action="store_true")
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="auto", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--topk", default="")
    ap.add_argument("--step-launches", type=int, default=0)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_beer.py measures the fused kernels and needs a CUDA device")
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
    problems = {}
    for pc in conf["problem_configs"].values():
        oc = pc["optimizer_config"]
        alg = {"dsgt": "dsgt", "choco_sgd": "choco", "beer": "beer"}[oc["alg_name"]]
        problems[alg if alg == "dsgt" else f"{alg}_{oc['compressor']}"] = pc
    for name, like in (("choco_sign", "choco_int8"), ("beer_none", "beer_int8")):
        problems[name] = copy.deepcopy(problems[like])
        problems[name]["optimizer_config"]["compressor"] = name.split("_")[1]
    problems["beer_none"]["optimizer_config"]["gamma"] = 1.0
    names = ["dsgt", "choco_int8", "choco_sign", "beer_none", "beer_int8", "beer_sign"]
    swept = ["choco_int8", "choco_sign", "beer_int8", "beer_sign"]
    for r in [float(x) for x in args.topk.split(",") if x]:
        for alg in ("choco", "beer"):
            name = f"{alg}_topk{r:g}"
            problems[name] = copy.deepcopy(problems[f"{alg}_int8"])
            problems[name]["optimizer_config"].update(compressor="topk", topk_ratio=r)
            names.append(name)
            swept.append(name)
    gammas = {}

    def build(name, dtype, rounds, eval_every, gamma=None):
        pc = copy.deepcopy(problems[name])
        pc["optimizer_config"]["outer_iterations"] = rounds
        if gamma is not None:
            pc["optimizer_config"]["gamma"] = gamma
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
              "bytes": {}, "accuracy": {}, "sweep": {}, "rounds": args.rounds, "warmup": args.warmup,
              "repeats": args.repeats, "multi_gpu": "not measured"}
    for dname in [d for d in args.dtypes.split(",") if d]:
        times = {a: [] for a in names}
        for _ in range(args.repeats):
            for name in names:
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
                record["bytes"].setdefault(dname, {})[name] = opt._program.eng.bytes_per_round()
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        record["speed_ms_per_round"][dname] = {"median": med, "all": times}
        print(f"{dname}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in names) + f"   (all {times})", flush=True)
        print(f"{dname}: bytes (row / pulled per round) "
              + "  ".join(f"{a} {b['row']}/{b['pulled']}" for a, b in record["bytes"][dname].items()), flush=True)

    if args.step_launches > 0:
        dts = [d for d in args.dtypes.split(",") if d]
        kernels = {}
        for alg, step_of in (("choco", lambda op: op.choco_step), ("beer", lambda op: op.beer_step)):
            for d, v in step_kernel_times(build, [n for n in names if n.startswith(alg + "_")
                                                  and n.split("_")[1] not in ("none", "sign")],
                                          dts, args.step_launches, step_of).items():
                kernels.setdefault(d, {}).update(v)
        record["step_kernel_ms"] = kernels

    for g in [float(x) for x in args.sweep.split(",") if x]:
        for name in swept:
            pr, opt = build(name, torch.float32, args.sweep_rounds, args.sweep_rounds, gamma=g)
            opt.train()
            record["sweep"].setdefault(name, {})[g] = top1(pr)
            print(f"sweep fp32 {name} gamma {g}: mean top-1 after {args.sweep_rounds} rounds {top1(pr):.4f}", flush=True)
            del pr, opt
    if args.gamma_from_sweep and record["sweep"]:
        for name, res in record["sweep"].items():
            gammas[name] = max(res, key=lambda g: (res[g], -list(res).index(g)))
        print(f"accuracy runs at the best swept gamma: {gammas}", flush=True)
    record["accuracy_gamma"] = {n: gammas.get(n, problems[n]["optimizer_config"].get("gamma")) for n in names}

    for dname in (args.accuracy_dtypes.split(",") if args.accuracy_rounds > 0 else []):
        acc = {}
        for name in names:
            pr, opt = build(name, DTYPES[dname], args.accuracy_rounds, args.accuracy_rounds, gamma=gammas.get(name))
            opt.train()
            acc[name] = top1(pr)
            del pr, opt
        record["accuracy"][dname] = acc
        print(f"{dname}: mean top-1 after {args.accuracy_rounds} rounds ({src}): "
              + "  ".join(f"{a} {acc[a]:.4f}" for a in names), flush=True)
    print("multi-GPU: not measured (one GPU)" if torch.cuda.device_count() < 2 else
          "multi-GPU: not measured by this script", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
