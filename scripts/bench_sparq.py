"""SPARQ-SGD: what an event-triggered round costs on the device, how often nodes trigger, the bytes the mixes really
pulled and the accuracy they bought, next to DSGD and CHOCO-SGD int8, on the dist_mnist_choco setup; a threshold sweep.

    python scripts/bench_sparq.py [--batch 64] [--dtype fp32] [--rounds 400] [--warmup 40] [--repeats 3]
                                  [--accuracy-rounds 2000] [--sweep] [--sweep-rounds 500]
                                  [--sweep-thresholds 1,10,...] [--only speed,accuracy]
                                  [--data-source synthetic_hard] [--out FILE.json]

The arms are those of ``experiments/dist_mnist_sparq.yaml`` (10-node cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), alpha0 0.005) on the fused sm_90a kernels.
  * speed: the arms alternate ``--repeats`` times in this process; each runs ``--warmup`` rounds, captures the CUDA
    graphs of the next ``--rounds`` rounds and times their replay with CUDA events (ms per round, median of repeats).
    On one GPU the pulls are L2 traffic: fewer pulled bytes are not claimed to be faster here;
  * accuracy: one run of ``--accuracy-rounds`` rounds per arm: the mean top-1 over nodes at the last evaluation, the
    fraction of node-rounds that triggered and the bytes the mixes pulled, counted on the device (``pulled_bytes``),
    against what CHOCO-SGD's mixes pull in as many rounds;
  * sweep (``--sweep``): SPARQ int8 (one local step) at every ``--sweep-thresholds`` value for ``--sweep-rounds``
    rounds: trigger fraction, pulled share and final mean top-1.
The card's name and power limit are printed in the same run.  Multi-GPU timings are not measured here.  Prints one JSON
line (and writes it to ``--out``).
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
from bench_dp import split_classes  # noqa: E402
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_sparq.yaml")
THRESHOLDS = "1,10,100,1000,10000,100000,1000000"


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--dtype", default="fp32", choices=list(DTYPES))
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--sweep-rounds", type=int, default=500)
    ap.add_argument("--sweep-thresholds", default=THRESHOLDS)
    ap.add_argument("--only", default="speed,accuracy")
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="synthetic_hard", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparq.py measures the fused kernels and needs a CUDA device")
    parts = set(args.only.split(","))
    dev = torch.device("cuda:0")
    dtype = DTYPES[args.dtype]
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    base = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}
    arms = list(base)
    train, src = load_mnist(args.data_dir, train=True, source=args.data_source)
    val, _ = load_mnist(args.data_dir, train=False, source=args.data_source)
    N = exp["graph"]["num_nodes"]
    _, cycle = graph_generation.generate_from_conf(dict(exp["graph"]))
    shards = split_classes(train, N)

    def build(problem, rounds, eval_every, **over):
        pc = copy.deepcopy(base[problem])
        pc["train_batch_size"] = args.batch
        oc = pc["optimizer_config"]
        oc.update(over, outer_iterations=rounds)
        pc["metrics_config"]["evaluate_frequency"] = eval_every
        pc["verbose_evals"] = False
        torch.manual_seed(0)
        m = exp["model"]
        model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
        pr = DistMNISTProblem(cycle, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
        opt = build_optimizer(pr, dev, oc)
        assert opt._use_engine(), f"{problem} does not run on the fused consensus kernels"
        return pr, opt

    def top1(pr):
        return round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1], dtype=torch.float64).mean()), 4)

    def traffic(opt):
        """(trigger fraction, bytes pulled, share of CHOCO-SGD's) of a finished SPARQ run."""
        trig = int(opt.pr.gather_rows(opt.triggers).sum())
        pulled, choco = opt.pulled_bytes(), opt.choco_bytes()
        return round(trig / (opt.k * N), 4), pulled, round(pulled / choco, 4)

    record = {"card": gpu, "data_source": src, "dtype": args.dtype, "graph": "cycle", "nodes": N, "batch": args.batch,
              "rounds": args.rounds, "warmup": args.warmup, "repeats": args.repeats,
              "accuracy_rounds": args.accuracy_rounds, "multi_gpu": "not measured",
              "thresholds": {a: base[a]["optimizer_config"].get("threshold") for a in arms}}
    if "speed" in parts:
        times = {a: [] for a in arms}
        record["bytes_per_round"], record["launches_per_round"] = {}, {}
        for _ in range(args.repeats):
            for name in arms:
                pr, opt = build(name, args.warmup + args.rounds, 10 ** 9)
                opt.run_rounds(args.warmup)
                opt.prepare_rounds(args.rounds)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0.record()
                opt.run_rounds(args.rounds)
                t1.record()
                torch.cuda.synchronize()
                eng = opt._program.eng
                eng.check()
                times[name].append(round(t0.elapsed_time(t1) / args.rounds, 4))
                record["launches_per_round"][name] = opt._program.launches_per_round()
                record["bytes_per_round"][name] = eng.bytes_per_round()
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        record["ms_per_round"] = {"median": med, "all": times}
        print("ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in arms) + f"   (all {times})", flush=True)
        print("bytes per round " + "  ".join(f"{a} {record['bytes_per_round'][a]}" for a in arms), flush=True)
    if "accuracy" in parts and args.accuracy_rounds > 0:
        record["top1"], record["trigger_fraction"], record["pulled_bytes"], record["pulled_share"] = {}, {}, {}, {}
        choco_pulled = None
        for name in arms:
            pr, opt = build(name, args.accuracy_rounds, 20)
            opt.train()
            record["top1"][name] = top1(pr)
            if opt.alg_name == "sparq_sgd":
                f, pulled, share = traffic(opt)
                record["trigger_fraction"][name], record["pulled_bytes"][name], record["pulled_share"][name] = \
                    f, pulled, share
            elif opt.alg_name == "choco_sgd":
                choco_pulled = record["pulled_bytes"][name] = \
                    opt._program.eng.bytes_per_round()["pulled"] * args.accuracy_rounds
            del pr, opt
        print(f"mean top-1 after {args.accuracy_rounds} {args.dtype} rounds ({src}) "
              + "  ".join(f"{a} {record['top1'][a]:.4f}" for a in arms), flush=True)
        print(f"CHOCO int8 pulled {choco_pulled} bytes; SPARQ " + "  ".join(
            f"{a}: triggered {record['trigger_fraction'][a]:.3f}, pulled {record['pulled_bytes'][a]} "
            f"({100 * record['pulled_share'][a]:.1f} %)" for a in record["trigger_fraction"]), flush=True)
    if args.sweep and args.sweep_rounds > 0:
        rows = record["sweep"] = []
        for c in [float(x) for x in args.sweep_thresholds.split(",") if x]:
            pr, opt = build("sparq_int8_low", args.sweep_rounds, 20, threshold=c)
            opt.train()
            f, pulled, share = traffic(opt)
            rows.append({"threshold": c, "trigger_fraction": f, "pulled_bytes": pulled, "pulled_share": share,
                         "top1": top1(pr)})
            print(f"sweep threshold {c}: triggered {f:.3f}, pulled {pulled} ({100 * share:.1f} % of CHOCO), "
                  f"top-1 {top1(pr)}", flush=True)
            del pr, opt
    print("multi-GPU: not measured (one GPU)", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
