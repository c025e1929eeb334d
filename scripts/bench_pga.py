"""Gossip-PGA: the cost of its two kinds of round and what the periodic average buys, on 10- and 32-node cycles with
the heterogeneous split.  Device time per round of DSGD, of Gossip-PGA's gossip round and of its global round, and of
DSGD on the complete graph in sum mode (the same fp64 reduction as a global round); bytes per round; the final accuracy
and consensus distance of DSGD, DSGT, Gossip-PGA at periods 2, 4 and 16 and local SGD at periods 4 and 16.

    python scripts/bench_pga.py [--nodes 10,32] [--batch 64] [--dtype fp32] [--rounds 400] [--warmup 40]
                                [--repeats 3] [--accuracy-rounds 2000] [--data-source synthetic_hard] [--out FILE.json]

The problems are those of ``experiments/dist_mnist_pga.yaml`` (a cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), DSGD's schedule alpha0 0.005 / mu 0.001 untuned, DSGT at alpha 0.005, on the fused sm_90a
kernels), at ``--nodes`` nodes.
  * speed: the four speed arms alternate ``--repeats`` times in this process; each builds its problem, runs
    ``--warmup`` rounds, captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA
    events (ms per round, the median over repeats).  ``pga_gossip`` has a period past the run, so every round is a
    gossip round and its early-returning ``pga_sum`` launch is the overhead over DSGD; ``pga_global`` has period 1,
    every round a global round;
  * bytes: from the engine (computed, not measured): ``pulled`` per gossip round, and for Gossip-PGA ``global_row``,
    the fp64 partial-sum row each rank contributes per global round;
  * accuracy: one run of ``--accuracy-rounds`` rounds per accuracy arm; the mean over nodes of the top-1 accuracy at
    the last evaluation, and the consensus distance sqrt(mean_i |theta_i - mean theta|^2) of the final models.
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

import networkx as nx
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
YAML = os.path.join(ROOT, "experiments", "dist_mnist_pga.yaml")
# speed arms: (base problem of the YAML, optimizer overrides, graph); None is the YAML's cycle.  "pga_gossip" never
# averages (period past the run): the gossip-round cost; "pga_global" averages every round: the global-round cost,
# against DSGD on the complete graph in sum mode, which does the same reduction
SPEED = {"dsgd": ("dsgd", {}, None),
         "pga_gossip": ("gossip_pga_p4", {"period": None}, None),
         "pga_global": ("gossip_pga_p4", {"period": 1}, None),
         "dsgd_complete_sum": ("dsgd", {}, "complete")}
ACCURACY = {"dsgd": ("dsgd", {}), "dsgt": ("dsgt", {}),
            "pga_p2": ("gossip_pga_p4", {"period": 2}), "pga_p4": ("gossip_pga_p4", {}),
            "pga_p16": ("gossip_pga_p16", {}),
            "local_sgd_p4": ("local_sgd_p4", {}), "local_sgd_p16": ("local_sgd_p4", {"period": 16})}


def split_classes(train, N):
    """The heterogeneous split of ``dist_mnist_ex`` for N <= 10 classes' worth of nodes; beyond that node i holds a
    share of class i mod 10 (the nodes of one class split its samples round-robin), so neighbors on the cycle still
    hold different classes."""
    if N <= 10:
        return split_hetero(train, N)
    shards = []
    for i in range(N):
        owners = list(range(i % 10, N, 10))
        idx = torch.nonzero(train.y == i % 10).flatten()
        shards.append(train.select(idx[owners.index(i)::len(owners)]))
    return shards


def consensus_distance(theta: torch.Tensor) -> float:
    t = theta.double()
    return float(((t - t.mean(0)) ** 2).sum(1).mean().sqrt())


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--nodes", default="10,32")
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
        raise SystemExit("bench_pga.py measures the fused kernels and needs a CUDA device")
    dev = torch.device("cuda:0")
    dtype = DTYPES[args.dtype]
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    train, src = load_mnist(args.data_dir, train=True, source=args.data_source)
    val, _ = load_mnist(args.data_dir, train=False, source=args.data_source)
    base = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}

    record = {"card": gpu, "data_source": src, "dtype": args.dtype, "graph": "cycle", "batch": args.batch,
              "rounds": args.rounds, "warmup": args.warmup, "repeats": args.repeats,
              "accuracy_rounds": args.accuracy_rounds, "per_run": {}, "multi_gpu": "not measured"}
    for N in [int(n) for n in args.nodes.split(",") if n]:
        _, cycle = graph_generation.generate_from_conf(dict(exp["graph"], num_nodes=N))
        shards = split_classes(train, N)

        def build(problem, over, graph, rounds, eval_every):
            pc = copy.deepcopy(base[problem])
            pc["train_batch_size"] = args.batch
            oc = pc["optimizer_config"]
            oc.update({k: (rounds + 1 if k == "period" and v is None else v) for k, v in over.items()})
            oc["outer_iterations"] = rounds
            pc["metrics_config"]["evaluate_frequency"] = eval_every
            torch.manual_seed(0)
            m = exp["model"]
            model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
            g = nx.complete_graph(N) if graph == "complete" else cycle
            pr = DistMNISTProblem(g, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
            opt = build_optimizer(pr, dev, oc)
            assert opt._use_engine(), f"{problem} does not run on the fused consensus kernels"
            return pr, opt

        key = f"N{N}_B{args.batch}"
        rec = record["per_run"][key] = {"nodes": N, "batch": args.batch, "ms_per_round": {}, "launches_per_round": {},
                                        "bytes_per_round": {}, "top1": {}, "consensus_distance": {}}
        times = {a: [] for a in SPEED}
        for _ in range(args.repeats):
            for name, (problem, over, graph) in SPEED.items():
                pr, opt = build(problem, over, graph, args.warmup + args.rounds, 10 ** 9)
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
        print(f"{key}: gossip-round overhead over DSGD {med['pga_gossip'] - med['dsgd']:+.4f} ms; global round against "
              f"complete-graph DSGD in sum mode {med['pga_global'] - med['dsgd_complete_sum']:+.4f} ms", flush=True)
        print(f"{key}: bytes per round (computed) " + "  ".join(f"{a} {b}" for a, b in rec["bytes_per_round"].items()),
              flush=True)
        if args.accuracy_rounds > 0:
            for name, (problem, over) in ACCURACY.items():
                pr, opt = build(problem, over, None, args.accuracy_rounds, args.accuracy_rounds)
                opt.train()
                rec["top1"][name] = round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1],
                                                                dtype=torch.float64).mean()), 4)
                rec["consensus_distance"][name] = float(f"{consensus_distance(pr.arena.theta[:, :pr.layout.n]):.4e}")
                del pr, opt
            print(f"{key}: mean top-1 after {args.accuracy_rounds} {args.dtype} rounds ({src}) "
                  + "  ".join(f"{a} {rec['top1'][a]:.4f}" for a in ACCURACY), flush=True)
            print(f"{key}: final consensus distance "
                  + "  ".join(f"{a} {rec['consensus_distance'][a]:.3e}" for a in ACCURACY), flush=True)
    print("multi-GPU: not measured (one GPU)" if torch.cuda.device_count() < 2 else
          "multi-GPU: not measured by this script", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
