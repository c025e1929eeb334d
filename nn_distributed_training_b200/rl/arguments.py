"""Command-line arguments of the centralized PPO entry point (reference: RL/arguments.py:21-23)."""
import argparse


def get_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--mode", dest="mode", type=str, default="train")             # train | test
    p.add_argument("--actor_model", dest="actor_model", type=str, default="")     # warm-start / test weights
    p.add_argument("--critic_model", dest="critic_model", type=str, default="")
    p.add_argument("--num_envs", type=int, default=16)
    p.add_argument("--total_timesteps", type=int, default=10_000_000)
    p.add_argument("--device", type=str, default="cpu")
    p.add_argument("--rollout", choices=("torch", "cuda"), default="torch")  # cuda: fused rollout kernel (--device cuda)
    p.add_argument("--update", choices=("torch", "cuda"), default="torch")   # cuda: fused PPO update kernels (--device cuda)
    p.add_argument("--render", type=str, default="")          # test mode: write a GIF of the first episode here
    p.add_argument("--out_dir", type=str, default="./trained")  # train mode: weights + reward curves
    p.add_argument("--ID", type=int, default=0)
    p.add_argument("--save_freq", type=int, default=10)
    p.add_argument("--seed", type=int, default=None)
    p.add_argument("--gae_lambda", type=float, default=None)  # GAE(lambda) advantages, lambda in [0, 1]
    return p.parse_args(argv)
