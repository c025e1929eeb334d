"""DSGD, CHOCO-SGD (compressor none / int8 / sign) and optionally PowerGossip on the PAPER MNIST setup: device time per round, bytes published
per row and pulled per round, and final accuracy.

    python scripts/bench_compression.py [--dtypes fp64,fp32] [--rounds 400] [--warmup 40] [--repeats 3]
                                        [--accuracy-rounds 2000] [--accuracy-dtypes fp32]
                                        [--sweep 0.1,0.3,0.5,0.8,1.0] [--sweep-rounds 500]
                                        [--data-source auto|mnist|synthetic|synthetic_hard] [--out FILE.json]
                                        [--topk 0.01,0.05] [--step-launches 2000] [--powergossip 1.0]

The problems are those of ``experiments/dist_mnist_choco.yaml`` (a 10-node cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), batch 64, on the fused sm_90a kernels), with ``choco_none`` added at the int8 problem's gamma.
  * speed: for each dtype the four configurations alternate ``--repeats`` times; each builds its problem, runs
    ``--warmup`` rounds, captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA
    events (ms per round, the median over repeats);
  * bytes: one published row per node and everything this process's nodes pull per round, from the engine;
  * accuracy: one run of ``--accuracy-rounds`` rounds per configuration and dtype; the mean over nodes of the top-1
    accuracy at the last evaluation;
  * ``--sweep``: the int8 and sign runs of ``--sweep-rounds`` rounds at each gamma (fp32), mean top-1 at the end;
  * ``--topk``: a ``choco_topk<ratio>`` configuration per ratio (the int8 problem with compressor topk), measured with
    the others; ``--step-launches``: the step kernel alone, int8 against each top-k ratio, timed with CUDA events over
    that many back-to-back launches replayed from one CUDA graph (ms per launch, per dtype).
  * ``--powergossip``: a ``powergossip`` configuration (rank-one compressed edge differences, the int8 problem's step
    schedule) at that gamma, measured with the others.
Without ``--topk`` and ``--powergossip`` the output is that of the four configurations above.
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
YAML = os.path.join(ROOT, "experiments", "dist_mnist_choco.yaml")


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
    ap.add_argument("--topk", default="")
    ap.add_argument("--step-launches", type=int, default=0)
    ap.add_argument("--powergossip", type=float, default=None, help="add PowerGossip at this gamma")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_compression.py measures the fused kernels and needs a CUDA device")
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
        problems["dsgd" if oc["alg_name"] == "dsgd" else "choco_" + oc["compressor"]] = pc
    problems["choco_none"] = copy.deepcopy(problems["choco_int8"])
    problems["choco_none"]["optimizer_config"]["compressor"] = "none"
    names = ["dsgd", "choco_none", "choco_int8", "choco_sign"]
    for r in [float(x) for x in args.topk.split(",") if x]:
        problems[f"choco_topk{r:g}"] = copy.deepcopy(problems["choco_int8"])
        problems[f"choco_topk{r:g}"]["optimizer_config"].update(compressor="topk", topk_ratio=r)
        names.append(f"choco_topk{r:g}")
    if args.powergossip is not None:
        pg = problems["powergossip"] = copy.deepcopy(problems["choco_int8"])
        oc = pg["optimizer_config"]
        pg["optimizer_config"] = {"alg_name": "powergossip", "gamma": args.powergossip, "alpha0": oc["alpha0"],
                                  "mu": oc["mu"], "outer_iterations": oc["outer_iterations"], "profile": False}
        names.append("powergossip")

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
        record["step_kernel_ms"] = step_kernel_times(build, [n for n in names if n.startswith("choco_")
                                                            and n.split("_")[1] not in ("none", "sign")],
                                                     [d for d in args.dtypes.split(",") if d], args.step_launches,
                                                     lambda op: op.choco_step)

    for g in [float(x) for x in args.sweep.split(",") if x]:
        for name in ("choco_int8", "choco_sign"):
            pr, opt = build(name, torch.float32, args.sweep_rounds, args.sweep_rounds, gamma=g)
            opt.train()
            record["sweep"].setdefault(name, {})[g] = top1(pr)
            print(f"sweep fp32 {name} gamma {g}: mean top-1 after {args.sweep_rounds} rounds {top1(pr):.4f}", flush=True)
            del pr, opt

    for dname in (args.accuracy_dtypes.split(",") if args.accuracy_rounds > 0 else []):
        acc = {}
        for name in names:
            pr, opt = build(name, DTYPES[dname], args.accuracy_rounds, args.accuracy_rounds)
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


def step_kernel_times(build, names, dtypes, launches, step_of):
    """The step kernel alone: ``launches`` back-to-back launches of it captured in one CUDA graph (each launch advances
    the round counter, so the problem's schedule covers two replays), the second replay timed with CUDA events; ms per
    launch per dtype and name."""
    out = {}
    for dname in dtypes:
        for name in names:
            pr, opt = build(name, DTYPES[dname], 2 * launches + 2, 10 ** 9)
            opt.run_rounds(1)
            torch.cuda.synchronize()
            step = step_of(opt._program.eng.op)
            graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
            with torch.cuda.stream(stream):
                step()                                   # once outside the capture: first-launch set-up
                torch.cuda.synchronize()
                with torch.cuda.graph(graph, stream=stream):
                    for _ in range(launches):
                        step()
            graph.replay()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            graph.replay()
            t1.record()
            torch.cuda.synchronize()
            opt._program.eng.check()
            ms = round(t0.elapsed_time(t1) / launches, 5)
            out.setdefault(dname, {})[name] = ms
            print(f"{dname} {name}: step kernel {ms * 1000:.2f} us per launch ({launches} launches in one graph)",
                  flush=True)
            del graph, pr, opt
    return out


if __name__ == "__main__":
    main()
