"""Cross-gradient gossip against DSGD, Exact Diffusion and DSGT on the 10-node PAPER cycle with the heterogeneous split.
Device time per round and per gradient evaluation, bytes pulled per round, the final consensus distance and the final
accuracy, and an equal-gradient-budget DSGD arm.

    python scripts/bench_cross_gradient.py [--nodes 10] [--batches 64] [--dtype fp32] [--rounds 400] [--warmup 40]
                                           [--repeats 3] [--accuracy-rounds 2000] [--data-source synthetic_hard]
                                           [--out FILE.json]

The problems are those of ``experiments/dist_mnist_cross_gradient.yaml`` (a cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), DSGD's step alpha0 0.005, mu 0.001, untuned, on the fused sm_90a kernels) with a cross_weight
0.5 arm added, Exact Diffusion at the same step and DSGT at the PAPER's alpha 0.005.
  * speed: the arms alternate ``--repeats`` times in this process; each builds its problem, runs ``--warmup`` rounds,
    captures the CUDA graphs of the next ``--rounds`` rounds, and times their replay with CUDA events (ms per round, the
    median over repeats).  A cross-gradient round launches 1 + dmax forward/backward passes per node (3 on a cycle), the
    others one: ms per gradient evaluation divides by the launched count;
  * bytes: everything this process's nodes pull per round, from the engine (computed, not measured);
  * accuracy: one run of ``--accuracy-rounds`` rounds per arm, and DSGD for (1 + dmax) times as many rounds (the same
    number of gradient evaluations as a cross-gradient run); the mean over nodes of the top-1 accuracy at the last
    evaluation, and the consensus distance sqrt(mean_i |theta_i - mean theta|^2) of the final models.
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
from bench_hsgd import consensus_distance, split_classes  # noqa: E402
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_cross_gradient.yaml")
WEIGHTS = (0.0, 0.5, 1.0)
NAMES = ["dsgd"] + [f"cross_gradient_w{w:g}" for w in WEIGHTS] + ["exact_diffusion", "dsgt"]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--nodes", default="10")
    ap.add_argument("--batches", default="64")
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
        raise SystemExit("bench_cross_gradient.py measures the fused kernels and needs a CUDA device")
    dev = torch.device("cuda:0")
    dtype = DTYPES[args.dtype]
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    train, src = load_mnist(args.data_dir, train=True, source=args.data_source)
    val, _ = load_mnist(args.data_dir, train=False, source=args.data_source)
    base = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}
    problems = {"dsgd": base["dsgd"]}
    for w in WEIGHTS:
        pc = problems[f"cross_gradient_w{w:g}"] = copy.deepcopy(base["cross_gradient_w1"])
        pc["problem_name"] = f"cross_gradient_w{w:g}"
        pc["optimizer_config"].update(cross_weight=w)
    for name, oc in (("exact_diffusion", {"alg_name": "exact_diffusion", "alpha0": 0.005, "mu": 0.001}),
                     ("dsgt", {"alg_name": "dsgt", "alpha": 0.005, "init_grads": True})):
        pc = problems[name] = copy.deepcopy(base["dsgd"])
        pc["problem_name"] = name
        pc["optimizer_config"] = dict(oc, outer_iterations=2000, profile=False)

    record = {"card": gpu, "data_source": src, "dtype": args.dtype, "graph": "cycle", "rounds": args.rounds,
              "grad_evals_per_round": {},
              "warmup": args.warmup, "repeats": args.repeats, "accuracy_rounds": args.accuracy_rounds, "per_run": {},
              "multi_gpu": "not measured"}
    for N, B in [(int(n), int(b)) for n in args.nodes.split(",") if n for b in args.batches.split(",") if b]:
        _, graph = graph_generation.generate_from_conf(dict(exp["graph"], num_nodes=N))
        shards = split_classes(train, N)

        def build(name, rounds, eval_every):
            pc = copy.deepcopy(problems[name])
            pc["train_batch_size"] = B
            pc["optimizer_config"]["outer_iterations"] = rounds
            pc["metrics_config"]["evaluate_frequency"] = eval_every
            torch.manual_seed(0)
            m = exp["model"]
            model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
            pr = DistMNISTProblem(graph, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
            opt = build_optimizer(pr, dev, pc["optimizer_config"])
            assert opt._use_engine(), f"{name} does not run on the fused consensus kernels"
            return pr, opt

        key = f"N{N}_B{B}"
        rec = record["per_run"][key] = {"nodes": N, "batch": B, "ms_per_round": {}, "ms_per_grad_eval": {},
                                        "bytes_pulled_per_round": {}, "top1": {}, "consensus_distance": {}}
        times = {a: [] for a in NAMES}
        for _ in range(args.repeats):
            for name in NAMES:
                pr, opt = build(name, args.warmup + args.rounds, 10 ** 9)
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
                rec["bytes_pulled_per_round"][name] = opt._program.eng.bytes_per_round()["pulled"]
                record["grad_evals_per_round"][f"{key}/{name}"] = opt._program.eng.grad_evals()
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        rec["ms_per_round"] = {"median": med, "all": times}
        launched = {a: record["grad_evals_per_round"][f"{key}/{a}"]["launched"] / N for a in NAMES}
        rec["ms_per_grad_eval"] = {a: round(med[a] / launched[a], 4) for a in NAMES}
        print(f"{key}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in NAMES) + f"   (all {times})", flush=True)
        print(f"{key}: ms/gradient evaluation " + "  ".join(f"{a} {rec['ms_per_grad_eval'][a]:.4f}" for a in NAMES),
              flush=True)
        print(f"{key}: bytes pulled per round (computed) "
              + "  ".join(f"{a} {b}" for a, b in rec["bytes_pulled_per_round"].items()), flush=True)
        if args.accuracy_rounds > 0:
            # the equal gradient budget: DSGD for as many rounds as a cross-gradient run launches gradients per node
            budget = int(launched["cross_gradient_w1"]) * args.accuracy_rounds
            problems["dsgd_equal_budget"] = copy.deepcopy(problems["dsgd"])
            arms = [(a, args.accuracy_rounds) for a in NAMES] + [("dsgd_equal_budget", budget)]
            rec["accuracy_rounds"] = dict(arms)
            for name, rounds in arms:
                pr, opt = build(name, rounds, rounds)
                opt.train()
                rec["top1"][name] = round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1],
                                                                dtype=torch.float64).mean()), 4)
                rec["consensus_distance"][name] = float(f"{consensus_distance(pr.arena.theta[:, :pr.layout.n]):.4e}")
                del pr, opt
            print(f"{key}: mean top-1 after {args.accuracy_rounds} {args.dtype} rounds ({src}; dsgd_equal_budget "
                  f"{budget}) " + "  ".join(f"{a} {v:.4f}" for a, v in rec["top1"].items()), flush=True)
            print(f"{key}: final consensus distance "
                  + "  ".join(f"{a} {v:.3e}" for a, v in rec["consensus_distance"].items()), flush=True)
    print("multi-GPU: not measured (one GPU)" if torch.cuda.device_count() < 2 else
          "multi-GPU: not measured by this script", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
