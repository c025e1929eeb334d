"""Generalized advantage estimation on the H100: what the GAE stage costs the advantage pass, and what it does to the
distributed-PPO reward curves.

    python scripts/bench_gae.py [--envs 16 256 4096] [--launches 200] [--repeats 3] [--out DIR]
    python scripts/bench_gae.py --rewards [--seeds 0 1 2] [--trainers cadmm dsgd dsgt] [--out DIR]

Timing: for each ``num_envs`` one batch of ``train_cadmm_multi``'s problem (3 predators, [12,64,64,64,1] critics,
50-cycle episodes) from the rollout kernel; then ``ops.ppo_update.advantages`` without GAE (critic pass +
normalisation, two launches) and with ``gae_lambda`` 0.95 (critic pass + GAE scan + normalisation, three launches),
timed with CUDA events over ``--launches`` calls after a warm-up, alternating, ``--repeats`` times.

Rewards (``--rewards``): ``train_{cadmm,dsgd,dsgt}_multi`` with ``--device cuda --rollout cuda --update cuda
--consensus cuda`` (their default 10 M steps, 16 worlds) at ``gae_lambda`` unset and 0.95 for each seed, as a table of
the mean reward of the first 10 and last 50 iterations and the best iteration.  The card's name and power limit are
printed by the same run.
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from nn_distributed_training_b200.ops import ppo_update  # noqa: E402
from nn_distributed_training_b200.rl.consensus_ppo import DSGDPPO, DSGTPPO, DiNNOPPO  # noqa: E402
from nn_distributed_training_b200.rl.train_common import common_conf, make_problem, parse_args  # noqa: E402

LAM = 0.95


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _events(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n * 1e3          # us per call


def time_advantages(E, launches, repeats):
    args = parse_args(["--num_envs", str(E), "--device", "cuda", "--rollout", "cuda", "--update", "cuda", "--seed", "0",
                       "--gae_lambda", str(LAM)])
    pr, _ = make_problem(args)
    pr.split_rollout_marl()
    b = pr._batch
    N, R = b["rtgs"].shape
    adv, ret = torch.empty_like(b["rtgs"]), torch.empty_like(b["rtgs"])
    g = ppo_update.GAE(rews=b["rews"], gamma=pr.gamma, lam=LAM, T=pr._episode_T, E=E, returns=ret)
    plain = lambda: ppo_update.advantages(pr.critics, b["obs"], b["rtgs"], out=adv)            # noqa: E731
    gae = lambda: ppo_update.advantages(pr.critics, b["obs"], b["rtgs"], out=adv, gae=g)       # noqa: E731
    for f in (plain, gae):
        for _ in range(20):
            f()
    torch.cuda.synchronize()
    t = {"plain": [], "gae": []}
    for _ in range(repeats):
        t["plain"].append(_events(plain, launches))
        t["gae"].append(_events(gae, launches))
    return dict(num_envs=E, N=N, R=R, T=pr._episode_T, launches=launches,
                plain_us=[round(x, 2) for x in t["plain"]], gae_us=[round(x, 2) for x in t["gae"]])


def _trainer(name, pr, args, h):
    """The trainer of ``train_{name}_multi`` with that script's configuration."""
    dev = torch.device(args.device)
    if name == "cadmm":
        return DiNNOPPO(pr, dev, dict(common_conf(args), rho_init=1.0, rho_scaling=1.0, primal_lr_start=h["lr"],
                                      primal_lr_finish=0.001, lr_decay_type="constant", persistant_primal_opt=False,
                                      primal_iterations=h["n_updates_per_iteration"], outer_iterations=10_000_000))
    if name == "dsgd":
        return DSGDPPO(pr, dev, dict(common_conf(args), alpha0=h["lr"], mu=0.0))
    return DSGTPPO(pr, dev, dict(common_conf(args), alpha_actor=h["lr"], alpha_critic=h["lr"], init_grads=False))


def reward_run(name, lam, seed, steps):
    argv = ["--device", "cuda", "--rollout", "cuda", "--update", "cuda", "--consensus", "cuda", "--seed", str(seed),
            "--no_writeout", "--max_rl_timesteps", str(steps)] + ([] if lam is None else ["--gae_lambda", str(lam)])
    args = parse_args(argv)
    pr, hyper = make_problem(args)
    tr = _trainer(name, pr, args, hyper)
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        tr.train()
    torch.cuda.synchronize()
    r = np.asarray(tr.avg_ep_rews)
    return dict(trainer=name, gae_lambda=lam, seed=seed, iterations=len(r), first10=round(float(r[:10].mean()), 2),
                last50=round(float(r[-50:].mean()), 2), max=round(float(r.max()), 2),
                wall_s=round(time.perf_counter() - t0, 1)), r


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[16, 256, 4096])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--rewards", action="store_true", help="run the reward comparison instead of the timing")
    ap.add_argument("--trainers", nargs="+", default=["cadmm", "dsgd", "dsgt"], choices=["cadmm", "dsgd", "dsgt"])
    ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1, 2])
    ap.add_argument("--steps", type=int, default=10_000_000)
    ap.add_argument("--out", default=None, help="write the rows (and the reward curves) here")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_gae.py needs a CUDA device")
    print("card:", card(), flush=True)
    rows, curves = [], {}
    if not a.rewards:
        for E in a.envs:
            rows.append(time_advantages(E, a.launches, a.repeats))
            print(json.dumps(rows[-1]), flush=True)
    else:
        for name in a.trainers:
            for lam in (None, LAM):
                for s in a.seeds:
                    row, r = reward_run(name, lam, s, a.steps)
                    rows.append(row)
                    curves[f"{name}_{lam}_{s}"] = r
                    print(json.dumps(row), flush=True)
        print("\n| trainer | gae_lambda | seed | first 10 | last 50 | max | wall s |\n|---|---|---|---|---|---|---|")
        for r in rows:
            print(f"| {r['trainer']} | {r['gae_lambda']} | {r['seed']} | {r['first10']} | {r['last50']} | {r['max']} | "
                  f"{r['wall_s']} |")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        tag = "rewards" if a.rewards else "timing"
        with open(os.path.join(a.out, f"bench_gae_{tag}.json"), "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)
        if curves:
            np.savez(os.path.join(a.out, "bench_gae_curves.npz"), **curves)


if __name__ == "__main__":
    main()
