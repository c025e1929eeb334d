"""SlowMo: the cost of its two kinds of round against Gossip-PGA's, and what the slow momentum buys, on cycles with the
heterogeneous split.  Device time per round of Gossip-PGA's and SlowMo's gossip rounds and global rounds at 10 and 32
nodes; bytes per round; the final accuracy and consensus distance of Gossip-PGA, local SGD and SlowMo over both, at
periods 4 and 16, slow_momentum 0, 0.5 and 0.7, and base momentum 0 and 0.9.

    python scripts/bench_slowmo.py [--nodes 10,32] [--accuracy-nodes 10] [--batch 64] [--dtype fp32] [--rounds 400]
                                   [--warmup 40] [--repeats 3] [--accuracy-rounds 2000] [--data-source synthetic_hard]
                                   [--out FILE.json]

The problems are those of ``experiments/dist_mnist_slowmo.yaml`` (a cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), DSGD's schedule alpha0 0.005 / mu 0.001 untuned, slow_lr 1, on the fused sm_90a kernels).
  * speed: the four speed arms alternate ``--repeats`` times in this process; each builds its problem, runs
    ``--warmup`` rounds, captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA
    events (ms per round, the median over repeats).  The ``_gossip`` arms have a period past the run, so every round is
    a gossip round and SlowMo's early-returning ``slowmo_outer`` launch is its overhead over Gossip-PGA; the ``_global``
    arms have period 1, every round a global round, where ``slowmo_outer`` runs the outer update;
  * bytes: from the engine (computed, not measured);
  * accuracy: at ``--accuracy-nodes`` nodes, one run of ``--accuracy-rounds`` rounds per arm; the mean over nodes of the
    top-1 accuracy at the last evaluation, and the consensus distance of the final models (bench_pga.py's).
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
from bench_pga import consensus_distance, split_classes  # noqa: E402
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_slowmo.yaml")
# speed arms: (base problem of the YAML, optimizer overrides); a period of None is one past the run (gossip rounds only)
SPEED = {"pga_gossip": ("gossip_pga_p4", {"period": None}), "slowmo_gossip": ("slowmo_p4", {"period": None}),
         "pga_global": ("gossip_pga_p4", {"period": 1}), "slowmo_global": ("slowmo_p4", {"period": 1})}


def accuracy_arms():
    """Gossip-PGA and local SGD at periods 4 and 16, and the SlowMo sweep over both bases."""
    arms = {"dsgd": ("dsgd", {})}
    for p in (4, 16):
        arms[f"pga_p{p}"] = ("gossip_pga_p4", {"period": p})
        arms[f"local_sgd_p{p}"] = ("local_sgd_p4", {"period": p})
    for base, problem in (("pga", "slowmo_p4"), ("local", "slowmo_local_p4")):
        for p in (4, 16):
            for bm in (0.0, 0.9):
                for sm in (0.0, 0.5, 0.7):
                    name = f"slowmo_{base}_p{p}_sm{sm}" + (f"_bm{bm}" if bm else "")
                    arms[name] = (problem, {"period": p, "slow_momentum": sm, "base_momentum": bm})
    return arms


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--nodes", default="10,32")
    ap.add_argument("--accuracy-nodes", default="10")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--dtype", default="fp32", choices=list(DTYPES))
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="synthetic_hard", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_slowmo.py measures the fused kernels and needs a CUDA device")
    dev = torch.device("cuda:0")
    dtype = DTYPES[args.dtype]
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    train, src = load_mnist(args.data_dir, train=True, source=args.data_source)
    val, _ = load_mnist(args.data_dir, train=False, source=args.data_source)
    base = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}
    acc_nodes = {int(n) for n in args.accuracy_nodes.split(",") if n}
    record = {"card": gpu, "data_source": src, "dtype": args.dtype, "graph": "cycle", "batch": args.batch,
              "rounds": args.rounds, "warmup": args.warmup, "repeats": args.repeats,
              "accuracy_rounds": args.accuracy_rounds, "per_run": {}, "multi_gpu": "not measured"}
    for N in sorted({int(n) for n in args.nodes.split(",") if n} | acc_nodes):
        _, cycle = graph_generation.generate_from_conf(dict(exp["graph"], num_nodes=N))
        shards = split_classes(train, N)

        def build(problem, over, rounds, eval_every):
            pc = copy.deepcopy(base[problem])
            pc["train_batch_size"] = args.batch
            oc = pc["optimizer_config"]
            oc.update({k: (rounds + 1 if k == "period" and v is None else v) for k, v in over.items()})
            oc["outer_iterations"] = rounds
            pc["metrics_config"]["evaluate_frequency"] = eval_every
            torch.manual_seed(0)
            m = exp["model"]
            model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
            pr = DistMNISTProblem(cycle, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
            opt = build_optimizer(pr, dev, oc)
            assert opt._use_engine(), f"{problem} does not run on the fused consensus kernels"
            return pr, opt

        key = f"N{N}_B{args.batch}"
        rec = record["per_run"][key] = {"nodes": N, "batch": args.batch, "ms_per_round": {}, "launches_per_round": {},
                                        "bytes_per_round": {}, "top1": {}, "consensus_distance": {}}
        if str(N) in args.nodes.split(","):
            times = {a: [] for a in SPEED}
            for _ in range(args.repeats):
                for name, (problem, over) in SPEED.items():
                    pr, opt = build(problem, over, args.warmup + args.rounds, 10 ** 9)
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
                    rec["launches_per_round"][name] = opt._program.launches_per_round()
                    rec["bytes_per_round"][name] = opt._program.eng.bytes_per_round()
                    del pr, opt
            med = {a: statistics.median(v) for a, v in times.items()}
            rec["ms_per_round"] = {"median": med, "all": times}
            print(f"{key}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in SPEED) + f"   (all {times})", flush=True)
            print(f"{key}: SlowMo over Gossip-PGA: gossip round {med['slowmo_gossip'] - med['pga_gossip']:+.4f} ms, "
                  f"global round {med['slowmo_global'] - med['pga_global']:+.4f} ms", flush=True)
            print(f"{key}: bytes per round (computed) " + "  ".join(f"{a} {b}" for a, b in rec["bytes_per_round"].items()),
                  flush=True)
        if N in acc_nodes and args.accuracy_rounds > 0:
            arms = accuracy_arms()
            for name, (problem, over) in arms.items():
                pr, opt = build(problem, over, args.accuracy_rounds, args.accuracy_rounds)
                opt.train()
                rec["top1"][name] = round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1],
                                                                dtype=torch.float64).mean()), 4)
                rec["consensus_distance"][name] = float(f"{consensus_distance(pr.arena.theta[:, :pr.layout.n]):.4e}")
                print(f"{key}: {name}: top-1 {rec['top1'][name]:.4f}  consensus distance "
                      f"{rec['consensus_distance'][name]:.3e}", flush=True)
                del pr, opt
    print("multi-GPU: not measured (one GPU)" if torch.cuda.device_count() < 2 else
          "multi-GPU: not measured by this script", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
