"""Time multi-agent PPO rollouts and whole DiNNO-PPO iterations for the three rollout paths.

    python scripts/bench_rl.py [--envs 16 256 4096] [--paths cpu cuda kernel] [--repeats 2]

Paths: ``cpu`` = torch rollout on the CPU, ``cuda`` = torch rollout on the GPU, ``kernel`` = the fused rollout kernel
(ops/csrc/tag_rollout.cu).  The problem is ``train_cadmm_multi``'s (3 predators, 1 prey, 8 obstacles, [12,64,64,64,5]
actors, 2000 steps per batch, 50 cycles per episode); an iteration is the trainer's loop body: rollout, advantages and
one DiNNO round of 5 primal steps.  Every timing ends in a device synchronise, follows a warm-up, and is repeated
``--repeats`` times so the spread shows.  The card's name and power limit are printed by the same run.
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


def bench(path, E, repeats, budget_s):
    dev = "cpu" if path == "cpu" else "cuda"
    args = parse_args(["--num_envs", str(E), "--device", dev, "--rollout", "cuda" if path == "kernel" else "torch",
                       "--seed", "0", "--no_writeout"])
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
        k[0] += 1

    iteration()                                           # warm-up: module loads, allocator, fused-kernel set-up
    pr.split_rollout_marl()
    t_roll = _timed(pr.split_rollout_marl, dev, 1)
    n_roll = max(1, min(200, int(budget_s / max(t_roll, 1e-6))))
    t_it = _timed(iteration, dev, 1)
    n_it = max(1, min(50, int(budget_s / max(t_it, 1e-6))))
    rows = []
    for r in range(repeats):
        rows.append(dict(path=path, num_envs=E, repeat=r, rollout_ms=1e3 * _timed(pr.split_rollout_marl, dev, n_roll),
                         iteration_ms=1e3 * _timed(iteration, dev, n_it), n_rollout=n_roll, n_iteration=n_it,
                         samples_per_rollout=int(pr.curr_obs[0].shape[0]) * pr.N))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[16, 256, 4096])
    ap.add_argument("--paths", nargs="+", default=["cpu", "cuda", "kernel"], choices=["cpu", "cuda", "kernel"])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--budget", type=float, default=2.0, help="seconds per timed window (at least one call)")
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    a = ap.parse_args(argv)
    if any(p != "cpu" for p in a.paths):
        if not torch.cuda.is_available():
            raise SystemExit("the cuda and kernel paths need a CUDA device")
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True)
        print(q.stdout.strip(), flush=True)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    print(f"cpu threads: {torch.get_num_threads()}", flush=True)
    rows = []
    for E in a.envs:
        for p in a.paths:
            rows += bench(p, E, a.repeats, a.budget)
    print("\n| num_envs | path | rollout ms | iteration ms |\n|---|---|---|---|")
    for E in a.envs:
        for p in a.paths:
            rs = [r for r in rows if r["num_envs"] == E and r["path"] == p]
            print(f"| {E} | {p} | {', '.join(f'{r['rollout_ms']:.3g}' for r in rs)} | "
                  f"{', '.join(f'{r['iteration_ms']:.3g}' for r in rs)} |")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
