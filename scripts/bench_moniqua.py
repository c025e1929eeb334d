"""Moniqua: what a round of modulo-quantized gossip costs on the device and what it does to accuracy, on the
hetero-ED MNIST setup, next to DSGD, Exact Diffusion and CHOCO-SGD's int8 rows; a 500-round theta_bound sweep; one
online-density run on the moving disk graph.

    python scripts/bench_moniqua.py [--batch 64] [--dtype fp32] [--rounds 400] [--warmup 40] [--repeats 3]
                                    [--kernel-launches 1000] [--accuracy-rounds 2000] [--sweep-rounds 500]
                                    [--sweep-bounds 0.005,0.01,...] [--density-rounds 400] [--only speed,accuracy,...]
                                    [--data-source synthetic_hard] [--out FILE.json]

The problems are those of ``experiments/dist_mnist_moniqua.yaml`` (10-node cycle, the heterogeneous class split,
MNISTConvNet(3, 5, 64), alpha0 0.005), with CHOCO-SGD int8 from ``experiments/dist_mnist_choco.yaml``, on the fused
sm_90a kernels.
  * speed: the arms alternate ``--repeats`` times in this process; each runs ``--warmup`` rounds, captures the CUDA
    graphs of the next ``--rounds`` rounds and times their replay with CUDA events (ms per round, median of repeats);
    then ``--kernel-launches`` launches of ``mq_step`` alone, captured as one graph and timed over one replay.  The
    bytes per row and pulled per round are the engine's ``bytes_per_round()``.  On one GPU the pulls are L2 traffic:
    a smaller row is not claimed to be faster here;
  * accuracy: one run of ``--accuracy-rounds`` rounds per arm; the mean top-1 over nodes at the last evaluation, the
    consensus distance sqrt(mean_i |theta_i - mean theta|^2) of the final models, the margin hits and the largest
    edge-gap ratio over the evaluation points;
  * sweep: every Moniqua arm at every ``--sweep-bounds`` theta_bound for ``--sweep-rounds`` rounds: margin hits,
    largest edge-gap ratio and final mean top-1;
  * density: ``experiments/dist_online_dense_moniqua.yaml`` through the online-density problem, ``--density-rounds``
    rounds, every arm: margin hits, largest edge-gap ratio and final validation loss.
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
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_algorithms import card  # noqa: E402
from bench_dp import consensus_distance, split_classes  # noqa: E402
from nn_distributed_training_b200.data.mnist import load_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.problems import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils import graph_generation  # noqa: E402
from nn_distributed_training_b200.utils.config import load_experiment  # noqa: E402

DTYPES = {"fp64": torch.float64, "fp32": torch.float32}
YAML = os.path.join(ROOT, "experiments", "dist_mnist_moniqua.yaml")
CHOCO_YAML = os.path.join(ROOT, "experiments", "dist_mnist_choco.yaml")
DENSITY_YAML = os.path.join(ROOT, "experiments", "dist_online_dense_moniqua.yaml")
MQ_ARMS = tuple(f"moniqua_{b}_{n}bit" for b in ("dsgd", "ed") for n in (2, 4, 8))
ARMS = ("dsgd", "exact_diffusion", "choco_int8") + MQ_ARMS
BOUNDS = "0.005,0.01,0.02,0.05,0.1,0.2,0.5,1.0"


def _report(pr, opt):
    gaps = pr.metrics.get("moniqua_edge_gap", [])
    hits = pr.metrics.get("moniqua_margin_hits")
    return (None if hits is None else int(hits.sum())), (round(max(gaps), 4) if gaps else None)


def density(rounds, bounds=None):
    """Every arm of the online-density YAML for ``rounds`` rounds through the runner's problem (with ``bounds``: every
    Moniqua arm at each of those theta_bound values instead of the YAML's); the results files go to a temporary
    directory."""
    from nn_distributed_training_b200.experiments import dist_online_dense_ex as dx
    import yaml
    with open(DENSITY_YAML) as f:
        conf = yaml.safe_load(f)
    if bounds:
        pcs = {}
        for key, pc in conf["problem_configs"].items():
            if pc["optimizer_config"]["alg_name"] != "moniqua":
                pcs[key] = pc
                continue
            for tb in bounds:
                q = copy.deepcopy(pc)
                q["problem_name"] = f"{pc['problem_name']}_tb{tb}"
                q["optimizer_config"]["theta_bound"] = tb
                pcs[f"{key}_tb{tb}"] = q
        conf["problem_configs"] = pcs
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        conf["experiment"]["output_metadir"] = tmp
        for pc in conf["problem_configs"].values():
            pc["optimizer_config"]["outer_iterations"] = rounds
        p = os.path.join(tmp, "c.yaml")
        with open(p, "w") as f:
            yaml.safe_dump(conf, f)
        cwd = os.getcwd()
        os.chdir(os.path.join(ROOT, "experiments"))
        try:
            dx.main(["dist_online_dense_ex.py", p])
        finally:
            os.chdir(cwd)
        for d in os.listdir(tmp):
            full = os.path.join(tmp, d)
            if not os.path.isdir(full):
                continue
            for name in conf["problem_configs"]:
                pname = conf["problem_configs"][name]["problem_name"]
                f = os.path.join(full, f"{pname}_results.pt")
                if os.path.exists(f):
                    r = torch.load(f, weights_only=False)
                    gaps = r.get("moniqua_edge_gap", [])
                    hits = r.get("moniqua_margin_hits")
                    out[pname] = {"validation_loss": float(torch.as_tensor(r["validation_loss"][-1]).double().mean()),
                                  "margin_hits": None if hits is None else int(hits.sum()),
                                  "max_edge_gap": round(max(gaps), 4) if gaps else None}
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--dtype", default="fp32", choices=list(DTYPES))
    ap.add_argument("--rounds", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=1000)
    ap.add_argument("--accuracy-rounds", type=int, default=2000)
    ap.add_argument("--sweep-rounds", type=int, default=500)
    ap.add_argument("--sweep-bounds", default=BOUNDS)
    ap.add_argument("--density-rounds", type=int, default=400)
    ap.add_argument("--density-bounds", default="", help="sweep the density arms over these theta_bound values")
    ap.add_argument("--only", default="speed,accuracy,sweep,density")
    ap.add_argument("--data-dir", default=os.path.join(ROOT, "..", "data"))
    ap.add_argument("--data-source", default="synthetic_hard", choices=["auto", "mnist", "synthetic", "synthetic_hard"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_moniqua.py measures the fused kernels and needs a CUDA device")
    parts = set(args.only.split(","))
    dev = torch.device("cuda:0")
    dtype = DTYPES[args.dtype]
    gpu = card()
    print(f"card: {gpu}", flush=True)

    conf = load_experiment(YAML, "mnist")
    exp = conf["experiment"]
    base = {pc["problem_name"]: pc for pc in conf["problem_configs"].values()}
    base["choco_int8"] = next(pc for pc in load_experiment(CHOCO_YAML, "mnist")["problem_configs"].values()
                              if pc["problem_name"] == "choco_int8")
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

    record = {"card": gpu, "data_source": src, "dtype": args.dtype, "graph": "cycle", "nodes": N, "batch": args.batch,
              "rounds": args.rounds, "warmup": args.warmup, "repeats": args.repeats,
              "kernel_launches": args.kernel_launches, "accuracy_rounds": args.accuracy_rounds,
              "theta_bound": {a: base[a]["optimizer_config"]["theta_bound"] for a in MQ_ARMS},
              "multi_gpu": "not measured"}
    if "speed" in parts:
        K = args.kernel_launches
        times = {a: [] for a in ARMS}
        kern = {a: [] for a in MQ_ARMS}
        record["bytes_per_round"], record["launches_per_round"] = {}, {}
        for _ in range(args.repeats):
            for name in ARMS:
                extra = K if name in MQ_ARMS else 0
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
                record["launches_per_round"][name] = opt._program.launches_per_round()
                record["bytes_per_round"][name] = eng.bytes_per_round()
                if extra:       # every mq_step advances the round counter, within the K extra rounds of the schedules
                    kern[name].append(round(graph_time(eng.op.mq_step, K) * 1e3, 3))
                    eng.check()
                del pr, opt
        med = {a: statistics.median(v) for a, v in times.items()}
        record["ms_per_round"] = {"median": med, "all": times}
        record["mq_step_us"] = {"median": {a: statistics.median(v) for a, v in kern.items()}, "all": kern}
        print("ms/round " + "  ".join(f"{a} {med[a]:.4f}" for a in ARMS) + f"   (all {times})", flush=True)
        print(f"mq_step us per launch over {K} graph-replayed launches " + "  ".join(
            f"{a} {statistics.median(v):.3f}" for a, v in kern.items()), flush=True)
        print("bytes per round " + "  ".join(f"{a} {record['bytes_per_round'][a]}" for a in ARMS), flush=True)
    if "accuracy" in parts and args.accuracy_rounds > 0:
        record["top1"], record["consensus_distance"], record["margin_hits"], record["max_edge_gap"] = {}, {}, {}, {}
        for name in ARMS:
            pr, opt = build(name, args.accuracy_rounds, 20)
            opt.train()
            record["top1"][name] = round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1],
                                                               dtype=torch.float64).mean()), 4)
            record["consensus_distance"][name] = float(f"{consensus_distance(pr.arena.theta[:, :pr.layout.n]):.4e}")
            if name in MQ_ARMS:
                record["margin_hits"][name], record["max_edge_gap"][name] = _report(pr, opt)
            del pr, opt
        print(f"mean top-1 after {args.accuracy_rounds} {args.dtype} rounds ({src}) "
              + "  ".join(f"{a} {record['top1'][a]:.4f}" for a in ARMS), flush=True)
        print("final consensus distance " + "  ".join(f"{a} {record['consensus_distance'][a]:.3e}" for a in ARMS),
              flush=True)
        print("margin hits / largest edge gap " + "  ".join(
            f"{a} {record['margin_hits'][a]} / {record['max_edge_gap'][a]}" for a in MQ_ARMS), flush=True)
    if "sweep" in parts and args.sweep_rounds > 0:
        sweep = record["sweep"] = {"rounds": args.sweep_rounds, "arms": {}}
        for name in MQ_ARMS:
            rows = sweep["arms"][name] = []
            for tb in [float(x) for x in args.sweep_bounds.split(",") if x]:
                pr, opt = build(name, args.sweep_rounds, 20, theta_bound=tb)
                opt.train()
                hits, gap = _report(pr, opt)
                top1 = round(float(torch.as_tensor(pr.metrics["top1_accuracy"][-1], dtype=torch.float64).mean()), 4)
                rows.append({"theta_bound": tb, "margin_hits": hits, "max_edge_gap": gap, "top1": top1})
                print(f"sweep {name} theta_bound {tb}: margin hits {hits}, largest edge gap {gap}, top-1 {top1}",
                      flush=True)
                del pr, opt
    if "density" in parts and args.density_rounds > 0:
        record["density"] = density(args.density_rounds, [float(x) for x in args.density_bounds.split(",") if x])
        print(f"online density ({args.density_rounds} rounds): {record['density']}", flush=True)
    print("multi-GPU: not measured (one GPU)", flush=True)
    line = json.dumps(record)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
