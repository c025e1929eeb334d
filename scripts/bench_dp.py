"""DP-DSGD / DECOR: the cost of node-level clipping and of the fp64 Box-Muller noise, and what the noise costs in
accuracy, on 10- and 32-node cycles with the heterogeneous split.  Device time per round of DSGD, clipped DSGD, local-DP
DSGD and DECOR; ``dp_norm`` and ``dp_step`` alone; the final accuracy and consensus distance of each arm with its two
epsilons.

    python scripts/bench_dp.py [--nodes 10,32] [--batch 64] [--dtype fp32] [--rounds 400] [--warmup 40]
                               [--repeats 3] [--kernel-launches 1000] [--accuracy-rounds 2000]
                               [--data-source synthetic_hard] [--out FILE.json]

The problems are those of ``experiments/dist_mnist_dp.yaml`` (a cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), DSGD's schedule alpha0 0.005 / mu 0.001 untuned, clip_norm 1, the multipliers calibrated to
node-level epsilon 8 against an eavesdropper over 2000 rounds), at ``--nodes`` nodes, on the fused sm_90a kernels.
  * speed: the four arms alternate ``--repeats`` times in this process; each builds its problem, runs ``--warmup``
    rounds, captures the CUDA graphs of the next ``--rounds`` rounds and times their replay with CUDA events (ms per
    round, the median over repeats);
  * kernels: after the timed rounds of the DECOR arm, ``--kernel-launches`` launches of ``dp_norm`` alone and of
    ``dp_step`` alone, each captured as one CUDA graph and timed over one replay (the schedules cover those rounds);
  * accuracy: one run of ``--accuracy-rounds`` rounds per arm; the mean over nodes of the top-1 accuracy at the last
    evaluation, the consensus distance sqrt(mean_i |theta_i - mean theta|^2) of the final models, and the accountant's
    epsilons (maximum over nodes) against an eavesdropper and against any observer.  The multipliers are the YAML's,
    calibrated for 10 nodes and 2000 rounds; the epsilons of other sizes are what the accountant reports for them.
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
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.experiments.dist_mnist_ex import split_hetero  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_dp.yaml")
ARMS = ("dsgd", "clipped_dsgd", "ldp_dsgd", "decor")


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
    ap.add_argument("--kernel-launches", type=int, default=1000)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="synthetic_hard", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_dp.py measures the fused kernels and needs a CUDA device")
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
              "kernel_launches": args.kernel_launches, "accuracy_rounds": args.accuracy_rounds, "per_run": {},
              "multi_gpu": "not measured"}
    for N in [int(n) for n in args.nodes.split(",") if n]:
        _, cycle = graph_generation.generate_from_conf(dict(exp["graph"], num_nodes=N))
        shards = split_classes(train, N)

        def build(problem, rounds, eval_every):
            pc = copy.deepcopy(base[problem])
            pc["train_batch_size"] = args.batch
            oc = pc["optimizer_config"]
            oc["outer_iterations"] = rounds
            pc["metrics_config"]["evaluate_frequency"] = eval_every
            torch.manual_seed(0)
            m = exp["model"]
            model = MNISTConvNet(m["num_filters"], m["kernel_size"], m["linear_width"], dtype=dtype)
            pr = DistMNISTProblem(cycle, model, torch.nn.NLLLoss(), shards, val, dev, pc, seed=0)
            opt = build_optimizer(pr, dev, oc)
            assert opt._use_engine(), f"{problem} does not run on the fused consensus kernels"
            return pr, opt

        def graph_time(fn, n):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(n):
                    fn()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            g.replay()
            t1.record()
            torch.cuda.synchronize()
            return t0.elapsed_time(t1) / n

        key = f"N{N}_B{args.batch}"
        rec = record["per_run"][key] = {"nodes": N, "batch": args.batch, "ms_per_round": {}, "launches_per_round": {},
                                        "bytes_per_round": {}, "kernel_ms": {}, "top1": {}, "consensus_distance": {},
                                        "epsilon_eavesdropper": {}, "epsilon_any_observer": {}}
        times = {a: [] for a in ARMS}
        kern = {"dp_norm": [], "dp_step": []}
        K = args.kernel_launches
        for _ in range(args.repeats):
            for name in ARMS:
                extra = 2 * K if name == "decor" else 0
                pr, opt = build(name, args.warmup + args.rounds + extra, 10 ** 9)
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
                rec["launches_per_round"][name] = opt._program.launches_per_round()
                rec["bytes_per_round"][name] = eng.bytes_per_round()
                if extra:
                    # dp_norm leaves the round counter alone; every dp_step advances it, within the 2 K extra rounds
                    # the schedules cover
                    kern["dp_norm"].append(round(graph_time(eng.op.dp_norm, K) * 1e3, 3))
                    kern["dp_step"].append(round(graph_time(eng.op.dp_step, K) * 1e3, 3))
                    eng.check()
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        rec["ms_per_round"] = {"median": med, "all": times}
        rec["kernel_ms"] = {"median_us": {k: statistics.median(v) for k, v in kern.items()}, "all_us": kern}
        print(f"{key}: ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in ARMS) + f"   (all {times})", flush=True)
        print(f"{key}: over DSGD: clipped {med['clipped_dsgd'] - med['dsgd']:+.4f} ms, local DP "
              f"{med['ldp_dsgd'] - med['dsgd']:+.4f} ms, DECOR {med['decor'] - med['dsgd']:+.4f} ms", flush=True)
        print(f"{key}: us per launch over {K} graph-replayed launches (DECOR): "
              + "  ".join(f"{k} {statistics.median(v):.3f}" for k, v in kern.items()) + f"   (all {kern})", flush=True)
        if args.accuracy_rounds > 0:
            for name in ARMS:
                pr, opt = build(name, args.accuracy_rounds, args.accuracy_rounds)
                opt.train()
                rec["top1"][name] = round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1],
                                                                dtype=torch.float64).mean()), 4)
                rec["consensus_distance"][name] = float(f"{consensus_distance(pr.arena.theta[:, :pr.layout.n]):.4e}")
                if name != "dsgd":
                    p = opt.privacy_record()
                    rec["epsilon_eavesdropper"][name] = p["epsilon_eavesdropper"]
                    rec["epsilon_any_observer"][name] = p["epsilon_any_observer"]
                del pr, opt
            print(f"{key}: mean top-1 after {args.accuracy_rounds} {args.dtype} rounds ({src}) "
                  + "  ".join(f"{a} {rec['top1'][a]:.4f}" for a in ARMS), flush=True)
            print(f"{key}: final consensus distance "
                  + "  ".join(f"{a} {rec['consensus_distance'][a]:.3e}" for a in ARMS), flush=True)
            print(f"{key}: epsilon (eavesdropper / any observer, delta 1e-5) "
                  + "  ".join(f"{a} {rec['epsilon_eavesdropper'][a]:.3f} / {rec['epsilon_any_observer'][a]:.3f}"
                              for a in ARMS[1:]), flush=True)
    print("multi-GPU: not measured (one GPU)" if torch.cuda.device_count() < 2 else
          "multi-GPU: not measured by this script", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
