"""Neighbor-exchange bandwidth sweep (BASELINE.json: bus GB/s vs 900 GB/s over a parameter-count sweep).

One graph node per GPU on a cycle; times the fused `dsgd_mix` kernel, which pulls both neighbors'
parameter rows over NVLink (P2P loads through the pointer table) and mixes them in registers, and —
as the baseline — an NCCL all_gather of the same rows followed by a torch matmul-free mix.
As in training, every `dsgd_mix` launch starts by announcing its round to the peers (a system fence and one
NVLink flag store per peer), so the fused time includes that announcement.  The round counter stays at 0,
so no rank ever waits for a peer.
Launch: torchrun --nproc-per-node G scripts/bench_exchange.py
Prints one JSON line per n on rank 0: device time (max over ranks), inbound GB/s per GPU."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist
from nn_distributed_training_b200.ops import load_ext
from nn_distributed_training_b200.parallel.context import DistContext
from nn_distributed_training_b200.parallel.symm import SymmetricBuffer

ctx = DistContext.from_env(use_cuda=True)
ext = load_ext(required=True)
dev, W, R = ctx.device, ctx.world_size, ctx.rank
sizes = [int(s) for s in os.environ.get("SIZES", "28544,1048576,16777216,67108864").split(",")]
nbrs = sorted({(R - 1) % W, (R + 1) % W} - {R})
for n in sizes:
    n_pad = (n + 127) // 128 * 128
    pub = SymmetricBuffer((2, 1, 1, n_pad), torch.float32, ctx)
    pub.local.normal_()
    theta = pub.local[0, 0].clone()
    flags = SymmetricBuffer((W,), torch.int32, ctx)
    flags.local.fill_(1 << 20)                      # neighbors "already published" every round we time
    d = max(1, len(nbrs))
    nbr_ptr = np.zeros((1, 1, d, 2, 1), dtype=np.int64); nbr_w = np.zeros((1, 1, d), np.float32); nbr_rank = -np.ones((1, 1, d), np.int32)
    for e, j in enumerate(nbrs):
        for par in range(2):
            nbr_ptr[0, 0, e, par, 0] = pub.peer_ptrs[j] + par * n_pad * 4
        nbr_w[0, 0, e] = 1.0 / 3; nbr_rank[0, 0, e] = j
    t = lambda a: torch.as_tensor(a, device=dev)
    T = dict(nbr_ptr=t(nbr_ptr), nbr_w=t(nbr_w), self_w=t(np.full((1, 1), 1.0 / 3, np.float32)), deg=t(np.full((1, 1), len(nbrs), np.int32)),
             nbr_rank=t(nbr_rank), round_ctr=torch.zeros(1, dtype=torch.int32, device=dev), sched=torch.zeros(8, device=dev),
             gid=torch.zeros(8, dtype=torch.int32, device=dev), done=torch.zeros(1, dtype=torch.int32, device=dev),
             err=torch.zeros(1, dtype=torch.int32, device=dev), peer_flag=t(np.asarray([flags.peer_ptrs[r] + 4 * R for r in range(W)], np.int64)))
    op = ext.ConsensusOpF32(dict(L=1, n_pad=n_pad, S=1, theta=theta.data_ptr(), grad_part=theta.data_ptr(), pub=pub.local.data_ptr(), C=1,
                                 pub_L=1, nbr_ptr=T["nbr_ptr"].data_ptr(), nbr_w=T["nbr_w"].data_ptr(), self_w=T["self_w"].data_ptr(),
                                 deg=T["deg"].data_ptr(), nbr_rank=T["nbr_rank"].data_ptr(), dmax=d, round_ctr=T["round_ctr"].data_ptr(),
                                 rho=T["sched"].data_ptr(), lr=T["sched"].data_ptr(), alpha=T["sched"].data_ptr(), graph_id=T["gid"].data_ptr(),
                                 flags=flags.local.data_ptr(), peer_flag=T["peer_flag"].data_ptr(), world=W, rank=R,
                                 done_ctr=T["done"].data_ptr(), err=T["err"].data_ptr()))
    def timed(fn, iters):
        for _ in range(3): fn()
        torch.cuda.synchronize(); ctx.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters): fn()
        e1.record(); torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1) / iters], device=dev, dtype=torch.float64)
        return float(ctx.all_reduce_max(ms).item())
    iters = 200 if n <= (1 << 20) else 20
    ms_fused = timed(op.dsgd_mix, iters)
    # NCCL baseline: all_gather every row, then mix with torch ops
    out = [torch.empty(n_pad, device=dev) for _ in range(W)]
    def nccl_mix():
        dist.all_gather(out, theta)
        acc = theta / 3
        for j in nbrs: acc = acc + out[j] / 3
        theta.copy_(acc)
    ms_nccl = timed(nccl_mix, iters) if W > 1 else float("nan")
    inbound = len(nbrs) * n_pad * 4
    if ctx.is_main:
        print(json.dumps({"n_params": n, "world": W, "neighbors": len(nbrs), "fused_us": ms_fused * 1e3,
                          "fused_inbound_GBps_per_gpu": inbound / (ms_fused * 1e-3) / 1e9,
                          "frac_of_770GBps_measured_peer_copy": inbound / (ms_fused * 1e-3) / 770e9,
                          "nccl_allgather_mix_us": ms_nccl * 1e3, "speedup_vs_nccl": ms_nccl / ms_fused,
                          "peer_mapping": pub.how}), flush=True)
    del op, pub, flags, theta, out
    torch.cuda.empty_cache(); ctx.barrier()
if dist.is_initialized():
    dist.destroy_process_group()
