"""Centralized PPO entry point (reference: RL/main.py): ``--mode train|test`` with optional
warm start from saved actor/critic weights (RL/main.py:35-38)."""
from __future__ import annotations

import sys

import torch

from .arguments import get_args
from .eval_policy import eval_policy
from .model import FFReLUNet
from .ppo import PPO
from .simple_tag import SimpleTagEnv


def make_env(num_envs=16, steps=200, device="cpu"):
    return SimpleTagEnv(num_envs=num_envs, num_good=1, num_adversaries=3, num_obstacles=8, max_cycles=steps, device=device)


def train(env, hyperparameters, actor_model, critic_model, total_timesteps):
    model = PPO(policy_class=FFReLUNet, env=env, **hyperparameters)
    if actor_model != "" and critic_model != "":
        print(f"Loading in {actor_model} and {critic_model}...", flush=True)
        model.actor.load_state_dict(torch.load(actor_model, map_location=env.device))
        model.critic.load_state_dict(torch.load(critic_model, map_location=env.device))
    elif actor_model != "" or critic_model != "":
        print("Error: Either specify both actor/critic models or none at all.")
        sys.exit(0)
    else:
        print("Training from scratch.", flush=True)
    model.learn(total_timesteps=total_timesteps)
    return model


def test(env, actor_model, render_to=None, backend="torch"):
    if actor_model == "":
        print("Didn't specify model file. Exiting.", flush=True)
        sys.exit(0)
    obs_dim = env.observation_spaces["adversary_0"].shape[0]
    policy = FFReLUNet([obs_dim, 64, 64, 64, 5])
    policy.load_state_dict(torch.load(actor_model, map_location=env.device))
    return eval_policy(policy.to(env.device), env, render_to=render_to or None, backend=backend)


def main(argv=None):
    args = get_args(argv)
    hyper = {"timesteps_per_batch": 2000, "max_timesteps_per_episode": 200, "gamma": 0.99,
             "n_updates_per_iteration": 10, "lr": 3e-4, "clip": 0.2, "out_dir": args.out_dir, "ID": args.ID,
             "save_freq": args.save_freq, "seed": args.seed, "rollout_backend": args.rollout,
             "update_backend": args.update, "gae_lambda": args.gae_lambda}
    env = make_env(args.num_envs, 200, args.device)
    if args.mode == "train":
        train(env, hyper, args.actor_model, args.critic_model, args.total_timesteps)
    else:
        test(env, args.actor_model, render_to=args.render, backend=args.rollout)


if __name__ == "__main__":
    main()
