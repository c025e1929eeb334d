"""Multi-process worker for BEER (launched by torch.distributed.run from test_distributed_beer.py).

Every rank hosts N/world graph nodes.  ``--delayed 0``: a few rounds; the gathered parameters, estimates, sums, tracker
and code rows must match a single-process run of the same problem (rank 0 recomputes it).  ``--delayed 1`` (GPUs):
every neighbor read is checked against its round tag and one rank is held back by spin kernels (BEER runs on a static graph only).  Both
channels of code rows are pulled from peer GPUs and decoded in the mix kernel, so the result must equal the
single-process one bit for bit."""
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
from nn_distributed_training_b200.optimizers import BEER  # noqa: E402
from nn_distributed_training_b200.parallel.context import DistContext  # noqa: E402
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem  # noqa: E402

CONF = {"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "compressor": "int8", "outer_iterations": 6, "profile": False}


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


def run(ctx, N, G, backend, delayed):
    R = 14 if delayed else CONF["outer_iterations"]
    conf = dict(copy.deepcopy(CONF), outer_iterations=R)
    extra = None
    if delayed:
        conf["debug_sequence_check"] = True
    pr = make(ctx, N, G, conf, backend, extra)
    opt = BEER(pr, ctx.device, copy.deepcopy(conf))
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
    else:
        opt.train()
    eng = getattr(getattr(opt, "_program", None), "eng", None)
    theta = pr.gather_rows(pr.arena.theta).cpu()
    if eng is not None:       # the fused run keeps the pending codes on the device: mirror them
        opt._program.sync_back()
    state = [pr.gather_rows(getattr(opt, n)).cpu() for n in BEER.STATE]
    ok = True
    if ctx.is_main:
        solo = DistContext.single(ctx.device)
        pr1 = make(solo, N, G, conf, backend, extra)
        opt1 = BEER(pr1, solo.device, copy.deepcopy(conf))
        if delayed:
            opt1.run_rounds(R)
        else:
            opt1.train()
        if getattr(opt1, "_program", None) is not None:
            opt1._program.sync_back()
        ref, ref_state = pr1.arena.theta.cpu(), [getattr(opt1, n).cpu() for n in BEER.STATE]
        rel = ((theta - ref).norm() / ref.norm()).item()
        # the consensus kernels are elementwise per node in a fixed neighbor order (BEER has no sum mode), and the gloo
        # path gathers the same codes: nothing depends on the placement
        ok = torch.equal(theta, ref) and all(torch.equal(x, y) for x, y in zip(state, ref_state))
        how = "" if eng is None else f" sum_mode={eng.sum_mode} distinct_graphs={len(eng.topos)}"
        print(f"[beer] world={ctx.world_size} delayed={delayed}{how} rel={rel:.2e} {'OK' if ok else 'MISMATCH'}", flush=True)
    ctx.barrier()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuda", type=int, default=0)
    ap.add_argument("--nodes", type=int, default=6)
    ap.add_argument("--graph", default="cycle")
    ap.add_argument("--delayed", type=int, default=0)
    args = ap.parse_args()
    ctx = DistContext.from_env(use_cuda=bool(args.cuda))
    N = args.nodes
    G = {"cycle": nx.cycle_graph(N), "wheel": nx.wheel_graph(N), "complete": nx.complete_graph(N)}[args.graph]
    ok = run(ctx, N, G, "fused" if args.cuda else "torch", bool(args.delayed))
    if ctx.is_main:
        print("DIST_RESULT", "PASS" if ok else "FAIL", flush=True)
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
