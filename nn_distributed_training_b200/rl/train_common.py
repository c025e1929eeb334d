"""Shared set-up of the three distributed-PPO entry points (reference: RL/dist_rl/train_{cadmm,dsgd,dsgt}_multi.py, which
hard-code these values; here they are the defaults of command-line flags)."""
import argparse

import networkx as nx

from .dist_ppo import DistPPOProblem
from .model import FFReLUNet
from .simple_tag import SimpleTagEnv

STEPS_PER_EPISODE = 200


def parse_args(argv=None, default_id=0):
    ap = argparse.ArgumentParser()
    ap.add_argument("--max_rl_timesteps", type=int, default=10_000_000)
    ap.add_argument("--num_envs", type=int, default=16, help="worlds stepped in lock-step by the batched environment")
    ap.add_argument("--device", default="cpu")
    ap.add_argument("--rollout", choices=("torch", "cuda"), default="torch",
                    help="cuda: each batch's rollout is one fused kernel launch (needs --device cuda)")
    ap.add_argument("--update", choices=("torch", "cuda"), default="torch",
                    help="cuda: advantages and each primal step's gradients of every predator are fused kernels "
                         "(needs --device cuda)")
    ap.add_argument("--consensus", choices=("torch", "cuda"), default="torch",
                    help="cuda: each iteration's consensus rounds run on the fused consensus kernels, replayed from one "
                         "CUDA graph with --update cuda (needs --device cuda)")
    ap.add_argument("--ID", type=int, default=default_id, help="suffix of the files written to --out_dir")
    ap.add_argument("--out_dir", default="./trained")
    ap.add_argument("--save_freq", type=int, default=10)
    ap.add_argument("--render", action="store_true", help="write an episode GIF every --render_every_i iterations")
    ap.add_argument("--render_every_i", type=int, default=10)
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--gae_lambda", type=float, default=None,
                    help="GAE(lambda) advantages and lambda-return critic targets, lambda in [0, 1] (default: "
                         "Monte-Carlo rewards-to-go)")
    ap.add_argument("--no_writeout", action="store_true")
    return ap.parse_args(argv)


def make_problem(args):
    """3 predators on a wheel graph chasing 1 heuristic prey among 8 fixed obstacles; actor / critic
    ``[obs, 64, 64, 64, act | 1]`` (reference: train_cadmm_multi.py:19-57)."""
    env = SimpleTagEnv(num_envs=args.num_envs, num_good=1, num_adversaries=3, num_obstacles=8,
                       max_cycles=STEPS_PER_EPISODE, device=args.device, seed=args.seed)
    hyper = {"timesteps_per_batch": 2000, "max_timesteps_per_episode": STEPS_PER_EPISODE, "gamma": 0.99,
             "n_updates_per_iteration": 5, "lr": 3e-4, "clip": 0.2, "render": bool(args.render),
             "render_every_i": args.render_every_i, "save_freq": args.save_freq, "seed": args.seed,
             "rollout_backend": args.rollout, "update_backend": args.update, "gae_lambda": args.gae_lambda}
    obs_dim = env.observation_spaces["adversary_0"].shape[0]
    act_dim = env.action_spaces["adversary_0"].shape[0]
    base_actor = FFReLUNet([obs_dim, 64, 64, 64, act_dim])
    base_critic = FFReLUNet([obs_dim, 64, 64, 64, 1])
    return DistPPOProblem(base_actor, base_critic, nx.wheel_graph(3), env, **hyper), hyper


def common_conf(args):
    return {"max_rl_timesteps": args.max_rl_timesteps, "ID": args.ID, "out_dir": args.out_dir,
            "writeout": not args.no_writeout, "consensus_backend": "fused" if args.consensus == "cuda" else "torch"}
