"""Time multi-agent PPO rollouts and whole DiNNO-PPO iterations for the three rollout paths and the two update paths.

    python scripts/bench_rl.py [--envs 16 256 4096] [--paths cpu cuda kernel] [--updates torch cuda]
                               [--consensus torch cuda] [--repeats 2]
    python scripts/bench_rl.py --profile OUT_DIR [--envs 16 4096] [--consensus cuda]

Paths: ``cpu`` = torch rollout on the CPU, ``cuda`` = torch rollout on the GPU, ``kernel`` = the fused rollout kernel
(ops/csrc/tag_rollout.cu).  Updates: ``torch`` = per-node autograd, ``cuda`` = the fused update kernels
(ops/csrc/ppo_update.cu; GPU paths only).  ``--consensus``: ``torch`` = the round as PyTorch ops from Python, ``cuda`` =
the fused consensus kernels (ops/csrc/consensus.cu) replayed from one CUDA graph per iteration (GPU paths only); without
the flag the trainer's default (torch) runs and the rows carry no consensus column.  The problem is ``train_cadmm_multi``'s (3 predators, 1 prey, 8 obstacles,
[12,64,64,64,5] actors, 2000 steps per batch, 50 cycles per episode); an iteration is the trainer's loop body: rollout,
advantages and one DiNNO round of 5 primal steps.  Every timing ends in a device synchronise and follows a warm-up; the
update (and consensus) paths of one (num_envs, path) are timed alternately, ``--repeats`` times, so the spread shows.  The card's name
and power limit are printed by the same run.

``--profile`` is a separate run (tracing slows the host): one ``torch.profiler`` trace per (num_envs, update) of the
kernel rollout path under OUT_DIR, and a split of an iteration's wall time into the rollout kernel, the update kernels,
the other device work and host gaps (with ``--consensus``: the consensus kernels as their own column), plus the grad kernel's achieved FLOP/s from ``grad_flops``.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from nn_distributed_training_b200.rl.consensus_ppo import DiNNOPPO  # noqa: E402
from nn_distributed_training_b200.rl.train_common import common_conf, make_problem, parse_args  # noqa: E402


def _sync(dev):
    if dev == "cuda":
        torch.cuda.synchronize()


def _timed(fn, dev, n):
    _sync(dev)
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    _sync(dev)
    return (time.perf_counter() - t0) / n


def grad_flops(actor_shape, critic_shape):
    """FLOP per sample of one primal step of the update: forward, dW and dH of every layer (no dH into the input)."""
    f = 0
    for shape in (actor_shape, critic_shape):
        mac = [a * b for a, b in zip(shape[:-1], shape[1:])]
        f += 2 * sum(mac) + 2 * sum(mac) + 2 * sum(mac[1:])
    return f


def setup(path, E, update, consensus=None):
    dev = "cpu" if path == "cpu" else "cuda"
    args = parse_args(["--num_envs", str(E), "--device", dev, "--rollout", "cuda" if path == "kernel" else "torch",
                       "--update", update, "--seed", "0", "--no_writeout"]
                      + (["--consensus", consensus] if consensus else []))
    pr, hyper = make_problem(args)
    conf = dict(common_conf(args), rho_init=1.0, rho_scaling=1.0, primal_lr_start=hyper["lr"], primal_lr_finish=0.001,
                lr_decay_type="constant", persistant_primal_opt=False, primal_iterations=hyper["n_updates_per_iteration"],
                outer_iterations=10 ** 6)
    tr = DiNNOPPO(pr, torch.device(dev), conf)
    k = [0]

    def iteration():
        pr.split_rollout_marl()
        pr.update_advantage()
        tr._consensus(k[0])
        pr.check_update()
        k[0] += 1

    iteration()                                           # warm-up: module loads, allocator, fused-kernel set-up
    pr.split_rollout_marl()
    return pr, iteration, dev


def bench(path, E, updates, repeats, budget_s, consensus=(None,)):
    runs = {(u, c): setup(path, E, u, c) for u in updates for c in consensus}
    n = {}
    for key, (pr, iteration, dev) in runs.items():
        t_roll = _timed(pr.split_rollout_marl, dev, 1)
        t_it = _timed(iteration, dev, 1)
        n[key] = (max(1, min(200, int(budget_s / max(t_roll, 1e-6)))), max(1, min(50, int(budget_s / max(t_it, 1e-6)))))
    rows = []
    for r in range(repeats):
        for (u, c), (pr, iteration, dev) in runs.items():  # update and consensus paths alternate within each repeat
            n_roll, n_it = n[(u, c)]
            row = dict(path=path, update=u, num_envs=E, repeat=r)
            if c is not None:
                row["consensus"] = c
            row.update(rollout_ms=1e3 * _timed(pr.split_rollout_marl, dev, n_roll),
                       iteration_ms=1e3 * _timed(iteration, dev, n_it), n_rollout=n_roll, n_iteration=n_it,
                       samples_per_rollout=int(pr.curr_obs[0].shape[0]) * pr.N)
            rows.append(row)
            print(json.dumps(rows[-1]), flush=True)
    return rows


CONSENSUS_KERNELS = ("local_sum", "dinno_update", "dsgd_mix", "dsgd_step", "dsgt_init", "dsgt_mix", "dsgt_track",
                     "consensus_metric", "inv_norm")


def profile(E, update, out_dir, n=5, consensus=None):
    from torch.profiler import ProfilerActivity, profile as tprofile
    pr, iteration, _ = setup("kernel", E, update, consensus)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        for _ in range(n):
            iteration()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) / n
    tag = f"_{consensus}" if consensus else ""
    prof.export_chrome_trace(os.path.join(out_dir, f"trace_E{E}_{update}{tag}.json"))
    split = dict(rollout_kernel=0.0, update_kernels=0.0, other_device=0.0)
    if consensus:
        split = dict(rollout_kernel=0.0, update_kernels=0.0, consensus_kernels=0.0, other_device=0.0)
    grad_us, grad_calls = 0.0, 0
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        if dt is None:
            dt = ev.cuda_time_total
        if ev.device_type.name != "CUDA" or dt <= 0:
            continue
        name = ev.key
        if "tag_rollout" in name:
            split["rollout_kernel"] += dt
        elif "ppo_" in name or "adv_norm" in name:
            split["update_kernels"] += dt
            if "ppo_grad_kernel" in name and "true>" in name:
                grad_us += dt
                grad_calls += ev.count
        elif consensus and any(k in name for k in CONSENSUS_KERNELS):
            split["consensus_kernels"] += dt
        else:
            split["other_device"] += dt
    row = {k: v / 1e3 / n for k, v in split.items()}           # ms per iteration
    row.update(num_envs=E, update=update, **({"consensus": consensus} if consensus else {}),
               iteration_ms_traced=1e3 * wall,
               host_gaps_ms=1e3 * wall - sum(v / 1e3 / n for v in split.values()))
    if grad_calls:
        samples = int(pr.curr_obs[0].shape[0]) * pr.N
        fl = grad_flops(pr.models[0].actor.shape, pr.models[0].critic.shape) * samples
        row.update(grad_kernel_us=grad_us / grad_calls, grad_flop_per_call=fl,
                   grad_tflops=fl / (grad_us / grad_calls * 1e-6) / 1e12)
    print(json.dumps(row), flush=True)
    return row


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[16, 256, 4096])
    ap.add_argument("--paths", nargs="+", default=["cpu", "cuda", "kernel"], choices=["cpu", "cuda", "kernel"])
    ap.add_argument("--updates", nargs="+", default=["torch"], choices=["torch", "cuda"])
    ap.add_argument("--consensus", nargs="+", default=None, choices=["torch", "cuda"],
                    help="consensus paths to time alternately (GPU paths only); default: the trainer's, no column")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--profile", default=None, help="profile the kernel rollout path with each update into this directory")
    ap.add_argument("--budget", type=float, default=2.0, help="seconds per timed window (at least one call)")
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    a = ap.parse_args(argv)
    if any(p != "cpu" for p in a.paths) or a.profile:
        if not torch.cuda.is_available():
            raise SystemExit("the cuda and kernel paths need a CUDA device")
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True)
        print(q.stdout.strip(), flush=True)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    print(f"cpu threads: {torch.get_num_threads()}", flush=True)
    if a.profile:
        os.makedirs(a.profile, exist_ok=True)
        rows = [profile(E, u, a.profile, consensus=c) for E in a.envs for u in a.updates for c in (a.consensus or [None])]
        with open(os.path.join(a.profile, "split.json"), "w") as f:
            json.dump(rows, f, indent=1)
        return
    rows = []
    cons = a.consensus or [None]
    for E in a.envs:
        for p in a.paths:
            rows += bench(p, E, [u for u in a.updates if p != "cpu" or u == "torch"], a.repeats, a.budget,
                          [c for c in cons if p != "cpu" or c in (None, "torch")])
    if a.consensus is None:
        print("\n| num_envs | path | update | rollout ms | iteration ms |\n|---|---|---|---|---|")
    else:
        print("\n| num_envs | path | update | consensus | rollout ms | iteration ms |\n|---|---|---|---|---|---|")
    for E in a.envs:
        for p in a.paths:
            for u in a.updates:
                for c in cons:
                    rs = [r for r in rows if r["num_envs"] == E and r["path"] == p and r["update"] == u
                          and r.get("consensus") == c]
                    if rs:
                        print(f"| {E} | {p} | {u} | {'' if c is None else c + ' | '}"
                              f"{', '.join(f'{r['rollout_ms']:.3g}' for r in rs)} | "
                              f"{', '.join(f'{r['iteration_ms']:.3g}' for r in rs)} |")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
