"""In-kernel phase timing of the batch-split MNIST training kernel (mnist_kernel<spb, 768, train> in
csrc/mnist.cu): with NNDT_STEP_PROF=1 every CTA stamps %globaltimer at its phase boundaries; prints the mean/max
duration of each phase over the CTAs of the last launch.

    python scripts/profile_round_phases.py [--nodes 10] [--rounds 200]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import bench  # noqa: E402


INNER = ["(images committed)", "conv+relu+pool (+W1 TMA wait)", "fc1 (mma)", "h reduce", "fc2", "softmax/loss",
         "fc2 grads, dh", "b1, da1 (mma), dW1 (mma) -> global", "conv-grad acc -> smem"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=200)
    args = ap.parse_args()
    from nn_distributed_training_b200.optimizers import DiNNO
    from nn_distributed_training_b200.parallel.context import DistContext
    os.environ["NNDT_STEP_PROF"] = "1"
    ctx = DistContext.single(torch.device("cuda:0"))
    pr = bench.build_problem(ctx, args.nodes, bench.opt_conf(4000), eval_every=10 ** 9, samples_per_node=22000)
    opt = DiNNO(pr, ctx.device, pr.conf["optimizer_config"])
    opt.run_rounds(args.rounds)
    torch.cuda.synchronize()
    t = pr.fused.step_prof.cpu().double()
    print(f"samples per CTA {pr.fused.spb}, CTAs per node {pr.fused.S}")
    rows = [("kernel start -> sampler chain done", 20, 21), ("image loads issued -> PDL wait returns", 21, 22),
            ("param staging + image commit", 22, 1)]
    prev = 1
    for j, n in enumerate(INNER[1:], start=2):
        rows.append((n, prev, j))
        prev = j
    rows.append(("conv-grad reduce + store", prev, 23))
    print(f"{'phase':44s} {'mean us':>9s} {'max us':>9s}")
    for n, a, b in rows:
        d = (t[:, b] - t[:, a]) / 1e3
        print(f"{n:44s} {d.mean().item():9.2f} {d.max().item():9.2f}")
    print(f"{'CTA lifetime':44s} {((t[:, 23] - t[:, 20]) / 1e3).mean().item():9.2f}")
    print(f"{'after the wait':44s} {((t[:, 23] - t[:, 22]) / 1e3).mean().item():9.2f}")
    print(f"{'first CTA start -> last CTA end':44s} {(t[:, 23].max() - t[:, 20].min()).item() / 1e3:9.2f}")


if __name__ == "__main__":
    main()
