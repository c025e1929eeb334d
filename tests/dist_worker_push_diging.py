"""Multi-process worker for Push-DIGing (launched by torch.distributed.run from test_distributed_push_diging.py).

Every rank hosts N/world graph nodes of a directed graph.  ``--delayed 0``: a few rounds; the gathered theta, u, w, y
and g_old must match a single-process run of the same problem (rank 0 recomputes it).  ``--delayed 1`` (GPUs): every in-neighbor
read is checked against its round tag and one rank is held back by spin kernels, so its peers run ahead as far as the
protocol lets them; the mix must also wait for the ranks that read a node's row in the previous round (its
out-neighbors), or a peer overwrites a buffer the slow rank still reads.  The graph ``switching`` changes every round, so
the previous round's readers come from another topology than the current in-neighbors.  The consensus kernels are
elementwise per node in a fixed neighbor order and the gloo path gathers the same rows, so the result must equal the
single-process one bit for bit."""
import argparse
import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dist_worker import METRICS  # noqa: E402
from dist_worker_sgp import SwitchingMNIST, graphs_of, _regular  # noqa: E402
from nn_distributed_training_b200.data.mnist import synthetic_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import PushDIGing  # noqa: E402
from nn_distributed_training_b200.parallel.context import DistContext  # noqa: E402

CONF = {"alg_name": "push_diging", "alpha": 0.05, "outer_iterations": 6, "profile": False}


def make(ctx, N, graphs, conf, backend):
    data = synthetic_mnist(200 * N, seed=3)
    val = synthetic_mnist(128, seed=4)
    shards = [data.select(torch.arange(i * 200, (i + 1) * 200)) for i in range(N)]
    # the same samples-per-CTA split in the distributed and the single-process run: identical fp32 gradient partials
    pconf = {"problem_name": "t", "train_batch_size": 32, "val_batch_size": 64, "metrics": METRICS, "samples_per_cta": 8,
             "metrics_config": {"evaluate_frequency": 3}, "optimizer_config": conf}
    torch.manual_seed(5)
    return SwitchingMNIST(graphs, MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, val, ctx.device, pconf, ctx=ctx,
                          backend=backend, seed=11)


def run(ctx, N, graphs, backend, delayed):
    R = 14 if delayed else CONF["outer_iterations"]
    conf = dict(copy.deepcopy(CONF), outer_iterations=R)
    if delayed:
        conf["debug_sequence_check"] = True
    pr = make(ctx, N, graphs, conf, backend)
    opt = PushDIGing(pr, ctx.device, copy.deepcopy(conf))
    if delayed:
        from nn_distributed_training_b200.ops import load_ext
        ext = load_ext(required=True)
        slow = ctx.world_size - 1
        for r in range(R):
            if ctx.rank == slow and r % 2 == 1:
                ext.spin(600_000)            # ~0.3 ms: many round times
            if ctx.rank == 0 and r % 3 == 2:
                ext.spin(300_000)
            opt.run_rounds(1)
        torch.cuda.synchronize()
        opt._program.eng.check()             # raises on a stale tag (err == 2) or a spin timeout
    else:
        opt.train()
    eng = getattr(getattr(opt, "_program", None), "eng", None)
    theta = pr.gather_rows(pr.arena.theta).cpu()
    if eng is not None:
        opt._program.sync_back()             # y lives in the published rows on the fused path
    state = [pr.gather_rows(opt.u).cpu(), pr.gather_rows(opt.w.view(-1, 1)).view(-1).cpu(),
             pr.gather_rows(opt.y).cpu(), pr.gather_rows(opt.g).cpu()]
    ok = True
    if ctx.is_main:
        solo = DistContext.single(ctx.device)
        pr1 = make(solo, N, graphs, conf, backend)
        opt1 = PushDIGing(pr1, solo.device, copy.deepcopy(conf))
        if delayed:
            opt1.run_rounds(R)
        else:
            opt1.train()
        if getattr(opt1, "_program", None) is not None:
            opt1._program.sync_back()
        ref, ref_state = pr1.arena.theta.cpu(), [opt1.u.cpu(), opt1.w.cpu(), opt1.y.cpu(), opt1.g.cpu()]
        rel = ((theta - ref).norm() / ref.norm()).item()
        ok = torch.equal(theta, ref) and all(torch.equal(x, y) for x, y in zip(state, ref_state))
        if len(graphs) > 1 or not _regular(graphs[0]):       # not doubly stochastic: w must have moved off 1
            ok = ok and not torch.all(ref_state[1] == 1.0)
        how = "" if eng is None else f" distinct_graphs={len(eng.topos)} notify_mask={eng.notify_mask:#x}"
        print(f"[push_diging] world={ctx.world_size} graphs={len(graphs)} delayed={delayed}{how} rel={rel:.2e} "
              f"w in [{ref_state[1].min():.3f}, {ref_state[1].max():.3f}] {'OK' if ok else 'MISMATCH'}", flush=True)
    ctx.barrier()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuda", type=int, default=0)
    ap.add_argument("--nodes", type=int, default=6)
    ap.add_argument("--graph", default="directed_cycle")
    ap.add_argument("--delayed", type=int, default=0)
    args = ap.parse_args()
    ctx = DistContext.from_env(use_cuda=bool(args.cuda))
    ok = run(ctx, args.nodes, graphs_of(args.graph, args.nodes), "fused" if args.cuda else "torch", bool(args.delayed))
    if ctx.is_main:
        print("DIST_RESULT", "PASS" if ok else "FAIL", flush=True)
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
