"""Roll out trained policies and report episodic returns (reference: RL/eval_policy.py and
RL/dist_rl/eval_policy.py:177-223).  Rendering: ``record=True`` keeps the positions ``[T, A, 2]`` of world 0 and
``save_rollout_gif`` turns them into an animation (the reference's pyglet window / vids/*.mp4)."""
from __future__ import annotations

import numpy as np
import torch

from .simple_tag import SimpleTagEnv, heuristic_prey_action


def rollout(actors, env: SimpleTagEnv, record=False, backend="torch"):
    """``actors``: one module (shared policy) or a list with one per predator.  Returns
    (episode return per world, episode length, optional positions).  ``backend="cuda"`` runs the deterministic
    episode as one kernel launch (ops/tag_rollout.py)."""
    if backend == "cuda":
        from ..ops import tag_rollout
        out = tag_rollout.rollout(env, actors, T=env.max_cycles, n_ep=1, gamma=1.0, cov_var=0.5, noise_scale=0.0,
                                  debug=record)
        traj = out["pos"][0, :, 0].cpu().numpy() if record else None
        return out["ep_returns"].float().cpu().numpy(), env.max_cycles, traj
    if backend != "torch":
        raise ValueError(f"backend must be 'torch' or 'cuda', not {backend!r}")
    shared = not isinstance(actors, (list, tuple, dict))
    obs_adv, obs_good = env.reset()
    total = torch.zeros(env.E, device=env.device)
    traj, t, done = [], 0, False
    while not done:
        acts = torch.zeros(env.E, env.A, 5, device=env.device, dtype=obs_adv.dtype)
        with torch.no_grad():
            for i in range(env.n_adv):
                net = actors if shared else actors[i]
                acts[:, i] = net(obs_adv[:, i])
        acts[:, env.n_adv:] = heuristic_prey_action(obs_good[:, 0], env.n_adv).unsqueeze(1)
        r_adv, _, done = env.step(acts)
        obs_adv, obs_good = env.observe()
        total += r_adv.sum(-1)
        t += 1
        if record:
            traj.append(env.pos[0].cpu().numpy().copy())
    return total.cpu().numpy(), t, (np.stack(traj) if record else None)


def save_rollout_gif(env: SimpleTagEnv, traj, out: str, size: int = 400, fps: int = 10) -> str:
    """Animated GIF of a recorded rollout (``traj [T, A, 2]``)."""
    frames = [env.render(size=size, pos=p) for p in traj]
    frames[0].save(out, save_all=True, append_images=frames[1:], duration=max(int(1000 / fps), 20), loop=0)
    return out


def eval_policy(actors, env: SimpleTagEnv, episodes=5, record=False, render_to=None, backend="torch"):
    """``render_to``: path of a GIF of the first episode (implies ``record``)."""
    rets = []
    for ep in range(episodes):
        ret, length, traj = rollout(actors, env, record=(record or render_to is not None) and ep == 0, backend=backend)
        if render_to is not None and ep == 0:
            save_rollout_gif(env, traj, render_to)
        rets.append(ret.mean())
        print(f"-------------------- Episode #{ep} --------------------\nEpisodic Length: {length}\n"
              f"Episodic Return: {ret.mean():.2f}\n------------------------------------------------------", flush=True)
    return float(np.mean(rets))


def load_distributed_actors(path, make_actor, n):
    """Load ``ppo_actors_tag_<alg>_<ID>_<k>.pth`` ({"actor0": state_dict, ...})."""
    sd = torch.load(path, map_location="cpu", weights_only=False)
    actors = []
    for i in range(n):
        a = make_actor()
        a.load_state_dict(sd[f"actor{i}"])
        actors.append(a)
    return actors
