"""Multi-process worker for ClippedGossip (launched by torch.distributed.run from test_distributed_clipped_gossip.py).

Every rank hosts N/world graph nodes; the Byzantine nodes are the first and the last node, so the first and the last
rank both host an attacker (and the ranks between, on GPUs, none: their step runs without the attack code).
``--delayed 0``: a few rounds on a static graph; the gathered parameters and published rows must match a
single-process run of the same problem (rank 0 recomputes it).  ``--delayed 1`` (GPUs): the graph changes every round
(link drops), every neighbor read at round start is checked against its round tag, one rank is held back by spin
kernels, and the peer-mapped result must equal the single-process one bit for bit: an ALIE attacker's reads of its
neighbors' rows after the mix must see the same rows as on one GPU."""
import argparse
import copy
import os
import sys

import networkx as nx
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dist_worker import METRICS  # noqa: E402
from nn_distributed_training_b200.data.mnist import synthetic_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import ClippedGossip  # noqa: E402
from nn_distributed_training_b200.parallel.context import DistContext  # noqa: E402
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem  # noqa: E402

CONF = {"alg_name": "clipped_gossip", "alpha0": 0.02, "mu": 0.001, "clip": "adaptive", "delta": 0.3,
        "outer_iterations": 6, "profile": False}


def make(ctx, N, G, conf, backend, extra=None):
    data = synthetic_mnist(200 * N, seed=3)
    val = synthetic_mnist(128, seed=4)
    shards = [data.select(torch.arange(i * 200, (i + 1) * 200)) for i in range(N)]
    # the same samples-per-CTA split in the distributed and the single-process run: identical fp32 gradient partials
    pconf = {"problem_name": "t", "train_batch_size": 32, "val_batch_size": 64, "metrics": METRICS, "samples_per_cta": 8,
             "metrics_config": {"evaluate_frequency": 3}, "optimizer_config": conf, **(extra or {})}
    torch.manual_seed(5)
    return DistMNISTProblem(G, MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, val, ctx.device, pconf, ctx=ctx,
                            backend=backend, seed=11)


def run(ctx, N, G, backend, delayed, clip, attack):
    R = 14 if delayed else CONF["outer_iterations"]
    conf = dict(copy.deepcopy(CONF), outer_iterations=R, clip=clip,
                byzantine={"nodes": [0, N - 1], "attack": attack, "scale": 2.0, "z": 1.0})
    extra = None
    if delayed:
        conf["debug_sequence_check"] = True
        extra = {"fault_injection": {"link_drop_prob": 0.45, "seed": 3, "from_round": 0, "to_round": R}}
    pr = make(ctx, N, G, conf, backend, extra)
    opt = ClippedGossip(pr, ctx.device, copy.deepcopy(conf))
    if delayed:
        from nn_distributed_training_b200.ops import load_ext
        ext = load_ext(required=True)
        slow = ctx.world_size - 1
        for r in range(R):
            if ctx.rank == slow and r % 2 == 1:
                ext.spin(600_000)
            if ctx.rank == 0 and r % 3 == 2:
                ext.spin(300_000)
            opt.run_rounds(1)
        torch.cuda.synchronize()
        opt._program.eng.check()
        opt._program.sync_back()
    else:
        opt.train()
    eng = getattr(getattr(opt, "_program", None), "eng", None)
    if eng is not None:
        assert (eng.t_attack is not None) == any(opt.attack), "attack codes on the wrong ranks"
    theta = pr.gather_rows(pr.arena.theta).cpu()
    pub = pr.gather_rows(opt.pub).cpu()
    ok = True
    if ctx.is_main:
        solo = DistContext.single(ctx.device)
        pr1 = make(solo, N, G, conf, backend, extra)
        opt1 = ClippedGossip(pr1, solo.device, copy.deepcopy(conf))
        if delayed:
            opt1.run_rounds(R)
            opt1._program.sync_back()
        else:
            opt1.train()
        ref, ref_pub = pr1.arena.theta.cpu(), opt1.pub.cpu()
        rel = ((theta - ref).norm() / ref.norm()).item()
        if eng is not None:
            # the kernels are elementwise per node in a fixed neighbor order, and the distance partials are per fixed
            # chunk of the row: nothing depends on the placement
            ok = torch.equal(theta, ref) and torch.equal(pub, ref_pub)
        else:
            bad = ((theta - ref).abs() > 2e-5 + 2e-3 * ref.abs()).float().mean().item()
            badp = ((pub - ref_pub).abs() > 2e-5 + 2e-3 * ref_pub.abs()).float().mean().item()
            ok = bad < 5e-3 and badp < 5e-3 and rel < 1e-2
        how = "" if eng is None else f" distinct_graphs={len(eng.topos)}"
        print(f"[clipped_gossip] world={ctx.world_size} delayed={delayed} clip={clip} attack={attack}{how} rel={rel:.2e} "
              f"{'OK' if ok else 'MISMATCH'}", flush=True)
    ctx.barrier()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuda", type=int, default=0)
    ap.add_argument("--nodes", type=int, default=6)
    ap.add_argument("--graph", default="cycle")
    ap.add_argument("--delayed", type=int, default=0)
    ap.add_argument("--clip", default="adaptive")
    ap.add_argument("--attack", default="alie")
    args = ap.parse_args()
    ctx = DistContext.from_env(use_cuda=bool(args.cuda))
    N = args.nodes
    G = {"cycle": nx.cycle_graph(N), "wheel": nx.wheel_graph(N), "complete": nx.complete_graph(N)}[args.graph]
    ok = run(ctx, N, G, "fused" if args.cuda else "torch", bool(args.delayed), args.clip, args.attack)
    if ctx.is_main:
        print("DIST_RESULT", "PASS" if ok else "FAIL", flush=True)
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
