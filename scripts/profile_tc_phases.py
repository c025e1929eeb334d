"""K-split cluster MNIST kernel (csrc/mnist_tc.cu): per-slot gradient error against PyTorch autograd and in-kernel phase timing
(%globaltimer stamps of every CTA of the last launch).

    NNDT_MNIST_TC=1 python scripts/profile_tc_phases.py [--nodes 10] [--rounds 100] [--split 0|1|2|4]
"""
import argparse
import os
import sys

os.environ.setdefault("NNDT_MNIST_TC", "1")
import networkx as nx
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import bench  # noqa: E402
from nn_distributed_training_b200.data.mnist import synthetic_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem  # noqa: E402

PHASES = ["sampler + image loads issued", "PDL wait", "TMA issue, small tensors, pixels -> fp32 planes", "conv + ReLU + pool -> A tile (hi/lo)",
          "W1 wait, MMA 1 (fc1)", "H partial -> smem, cluster sync 1", "reduce-scatter, fc2, loss, dz, dh, fc2 grads",
          "cluster sync 2", "fc2-grad reduce (1/6), gather dH, re-swizzle W", "MMA 2 (da1) | re-swizzle A; re-swizzle dH",
          "MMA 3 issue | da1 epilogue", "conv grads (under MMA 3) -> rank 0", "MMA 3 wait, dW1 epilogue -> global",
          "cluster sync 3, conv-grad sum (rank 0), exit"]
# MS <= 32 pushes H, dH and the fc2 shares (st.async): the sync rows are mbarrier waits, the reduce and gather row is empty and
# the fc2-grad reduce runs on the GEMM 3 warps before GEMM 3
PHASES64 = ["sampler, image rows -> smem (fp64)", "PDL wait", "W1 copies issued, conv weights + w2 (L2)",
            "conv + ReLU + pool -> A tile (fp64), W1 copy wait", "GEMM 1 (fc1 partial, DMMA), H pushes",
            "cluster sync 1 | H pushes wait", "head: warp per sample (H sum, fc2, loss, dz, dh), fc2 grads",
            "cluster sync 2 | dH pushes wait", "fc2-grad reduce (1/4), gather dH (MS = 64)",
            "GEMM 2 (da1, DMMA) -> registers", "da1 -> smem (over W)", "GEMM 3 (dW1, warps 16-19) -> global | conv grads",
            "bias warp, conv grads still running after GEMM 3 -> rank 0", "cluster sync 3, conv-grad sum (rank 0), exit"]


def slot_errors(B):
    conf = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}
    out = []
    probs = {}
    for backend in ("fused", "torch"):
        torch.manual_seed(0)
        data = synthetic_mnist(450, seed=3)
        val = synthetic_mnist(200, seed=4)
        shards = [data.select(torch.arange(i * 150, (i + 1) * 150)) for i in range(3)]
        pconf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": ["validation_loss"],
                 "metrics_config": {"evaluate_frequency": 1000}, "optimizer_config": conf}
        probs[backend] = DistMNISTProblem(nx.cycle_graph(3), MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, val, "cuda:0",
                                          pconf, backend=backend, seed=7)
    f, r = probs["fused"], probs["torch"]
    r.arena.theta.copy_(f.arena.theta)
    print(f"kernel: {f.fused.kernel_name}")
    for step in range(2):
        lf, lr = f.compute_grads().clone(), r.compute_grads().clone()
        print(f"step {step}: loss fused {lf.tolist()} ref {lr.tolist()}")
        for s in f.arena.layout.slots:
            a = f.arena.grad[:, s.offset: s.offset + s.numel]
            b = r.arena.grad[:, s.offset: s.offset + s.numel]
            rel = ((a - b).norm() / b.norm().clamp_min(1e-20)).item()
            print(f"   {s.name:14s} |ref| {b.norm().item():.3e} |fused| {a.norm().item():.3e} rel err {rel:.2e}")


def phases(nodes, rounds, dtype="fp32"):
    from nn_distributed_training_b200.optimizers import DiNNO
    from nn_distributed_training_b200.parallel.context import DistContext
    os.environ["NNDT_STEP_PROF"] = "1"
    ctx = DistContext.single(torch.device("cuda:0"))
    pr = bench.build_problem(ctx, bench._cycle(nodes), bench.opt_conf(4000), 10 ** 9, dtype=dtype)
    opt = DiNNO(pr, ctx.device, pr.conf["optimizer_config"])
    opt.run_rounds(rounds)
    torch.cuda.synchronize()
    t = pr.fused.step_prof.cpu().double()
    print(f"kernel: {pr.fused.kernel_name}; {t.shape[0]} CTAs")
    print(f"{'phase':58s} {'mean us':>9s} {'max us':>9s}")
    names = PHASES64 if dtype == "fp64" else PHASES
    last = len(names)
    for i, n in enumerate(names):
        d = (t[:, i + 1] - t[:, i]) / 1e3
        print(f"{n:58s} {d.mean().item():9.2f} {d.max().item():9.2f}")
    print(f"{'CTA lifetime':58s} {((t[:, last] - t[:, 0]) / 1e3).mean().item():9.2f}")
    print(f"{'after the PDL wait':58s} {((t[:, last] - t[:, 2]) / 1e3).mean().item():9.2f}")
    print(f"{'first CTA start -> last CTA end':58s} {(t[:, last].max() - t[:, 0].min()).item() / 1e3:9.2f}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=100)
    ap.add_argument("--split", type=int, default=0)
    args = ap.parse_args()
    if args.split:
        os.environ["NNDT_TC_SPLIT"] = str(args.split)
    torch.backends.cudnn.allow_tf32 = False       # the autograd reference must be fp32-accurate (cuDNN picks TF32 convs otherwise)
    slot_errors(64)
    slot_errors(24)
    phases(args.nodes, args.rounds)
    phases(args.nodes, args.rounds, "fp64")
