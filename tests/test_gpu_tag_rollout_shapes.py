"""The fused rollout kernel (ops/csrc/tag_rollout.cu) at every instantiation, launch plan and shape edge, against the
float64 replay oracle with the yardsticks of tests/tag_rollout_oracle.py (fp64: 10x the oracle's one-ulp-``pos0``
divergence and 1e-12 on the first two cycles; fp32: 4x torch fp32).

The cases reach all eight launches (fp32 / fp64 x 1 / 4 worlds per register block x actors staged in shared memory /
read in place), 1, 2, 3, 4 and 28 worlds per CTA with a partial last CTA, 1 + 1, 1 + 7 and 7 + 1 agents, 0 and 8
obstacles, 1-layer, width-1 and 5 x 64 actors, one actor shared by every predator and ``actor_of = [0, 1, 0]``, T = 1
and three episodes.  Every output, including the final state of every world, is poisoned with NaN and sits between
guard values.  One world run under different plans gives the same bits.
"""
import copy

import pytest
import torch

from nn_distributed_training_b200.ops import tag_rollout
from nn_distributed_training_b200.rl import FFReLUNet
from kernel_oracles import Guarded
from tag_rollout_oracle import COV, GAMMA, check_fp64, fp32_ratio, tag_env

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32 = torch.float64, torch.float32

# id: (dtype, env config, actor hidden layers, sharing, n_ep, T, plan (wpb, stage, rw) on 132 SMs with 227 KB)
CASES = {
    "fp64-rw1-staged-3ep": (F64, dict(E=16, n_adv=3, n_good=1, n_obst=8), (16,), "010", 3, 8, (1, 1, 1)),
    "fp32-rw1-staged-3ep": (F32, dict(E=16, n_adv=3, n_good=1, n_obst=8), (16,), "010", 3, 8, (1, 1, 1)),
    "fp64-wpb2-1v7-width1": (F64, dict(E=200, n_adv=1, n_good=7, n_obst=0), (1,), "own", 1, 6, (2, 1, 1)),
    "fp32-wpb3-T1-one-layer": (F32, dict(E=150, n_adv=3, n_good=1, n_obst=8), (), "shared", 2, 1, (3, 1, 1)),
    "fp64-rw4-staged-1v1-partial": (F64, dict(E=401, n_adv=1, n_good=1, n_obst=0), (32,), "own", 1, 6, (4, 1, 4)),
    "fp32-rw4-staged-1v1-partial": (F32, dict(E=401, n_adv=1, n_good=1, n_obst=0), (32,), "own", 1, 6, (4, 1, 4)),
    "fp64-rw1-inplace-7v1": (F64, dict(E=16, n_adv=7, n_good=1, n_obst=8), (64,) * 4, "own", 1, 4, (1, 0, 1)),
    "fp32-rw1-inplace-7v1": (F32, dict(E=16, n_adv=7, n_good=1, n_obst=8), (64,) * 4, "own", 1, 4, (1, 0, 1)),
    "fp32-rw4-inplace-7v1-partial": (F32, dict(E=401, n_adv=7, n_good=1, n_obst=8), (64,) * 4, "own", 1, 4, (4, 0, 4)),
    # 32 worlds of 7 fp64 predators need 242 KB even with the actors in place: the plan shrinks to 28 per CTA
    "fp64-rw4-inplace-shrink-28": (F64, dict(E=4100, n_adv=7, n_good=1, n_obst=0), (64,) * 4, "own", 1, 3, (28, 0, 4)),
}


def h100_sxm():
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count == 132 and p.shared_memory_per_block_optin == 227 * 1024


def actors_for(env, hidden, sharing, dtype, seed=1):
    """``own``: one actor per predator; ``shared``: one module for all; ``010``: predators 0 and 2 share actor 0."""
    torch.manual_seed(seed)
    d0 = env.observation_spaces["adversary_0"].shape[0]
    make = lambda: FFReLUNet([d0, *hidden, 5], dtype=dtype).to(DEV)          # noqa: E731
    if sharing == "shared":
        return [make()] * env.n_adv
    if sharing == "010":
        a, b = make(), make()
        return [a, b, a]
    return [make() for _ in range(env.n_adv)]


def poisoned(env, n_ep, T):
    """NaN-filled ``rollout`` outputs between guard values: every output of a debug rollout."""
    N, E, A, d0 = env.n_adv, env.E, env.A, env.observation_spaces["adversary_0"].shape[0]
    R = n_ep * T * E
    shapes = dict(obs=(N, R, d0), acts=(N, R, 5), log_probs=(N, R), rtgs=(N, R), ep_returns=(n_ep * E,),
                  final_pos=(n_ep, E, A, 2), final_vel=(n_ep, E, A, 2), eps=(N, R, 5), pos=(n_ep, T, E, A, 2))
    g = Guarded(list(shapes.values()), env.dtype, DEV)
    return g, dict(zip(shapes, g.views))


@pytest.mark.parametrize("case", list(CASES))
def test_rollout_against_the_oracle(case):
    dtype, cfg, hidden, sharing, n_ep, T, want = CASES[case]
    cfg = dict(cfg, max_cycles=200, dtype=dtype)
    env = tag_env(**cfg)
    actors = actors_for(env, hidden, sharing, dtype)
    plan = tag_rollout.launch_plan(env, actors, T, n_ep)
    if h100_sxm():
        assert (plan["wpb"], plan["stage"], plan["rw"]) == want, plan
    guard, out = poisoned(env, n_ep, T)
    if dtype == F64:
        res, worst = check_fp64(cfg, actors, n_ep, T, out=out)
    else:
        res, worst = fp32_ratio(cfg, actors, T, n_ep, out=out)
    guard.assert_guards(case)
    for k, v in res.items():
        assert v.data_ptr() == out[k].data_ptr() and not v.isnan().any(), k
    kind = "error / bound" if dtype == F64 else "error / torch fp32 error"
    print(f"tag_rollout {case}: plan {plan}; worst {kind} {worst:.3g}")


def test_plan_coverage():
    """The cases reach all eight (dtype, RW, stage) launches, 1, 2, 3, 4 and 28 worlds per CTA and partial last CTAs
    under RW = 4."""
    if not h100_sxm():
        pytest.skip("the expected plans are those of 132 SMs with 227 KB of opt-in shared memory")
    combos, wpbs, partial_rw4 = set(), set(), False
    for dtype, cfg, hidden, sharing, n_ep, T, _ in CASES.values():
        env = tag_env(**dict(cfg, dtype=dtype))
        p = tag_rollout.launch_plan(env, actors_for(env, hidden, sharing, dtype), T, n_ep)
        combos.add((dtype, p["rw"], p["stage"]))
        wpbs.add(p["wpb"])
        partial_rw4 |= p["rw"] == 4 and (n_ep * env.E) % p["wpb"] != 0
    assert len(combos) == 8, combos
    assert {1, 2, 3, 4, 28} <= wpbs and partial_rw4


@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_one_world_is_bitwise_equal_under_every_plan(dtype):
    """Episode 0 of E = (SM count) worlds, with 1, 2, 3, 4 and 8 episodes: 1, 2, 3, 4 and 8 worlds per CTA, RW 1 and 4,
    and (fp64, two 5 x 64 actors) staged and in-place weights.  Same key, index and pos0: every output of episode 0
    must be the same bits, since each world's arithmetic and noise counters do not depend on the grid."""
    E = torch.cuda.get_device_properties(0).multi_processor_count
    T = 6
    cfg = dict(E=E, n_adv=3, n_good=1, n_obst=8, dtype=dtype)
    env = tag_env(**cfg)
    actors = actors_for(env, (64,) * 4, "010", dtype)
    pos0 = tag_rollout.reset_positions(tag_env(**cfg), 8)
    base, plans = None, []
    for n_ep in (1, 2, 3, 4, 8):
        plans.append(tag_rollout.launch_plan(env, actors, T, n_ep))
        out = tag_rollout.rollout(env, actors, T=T, n_ep=n_ep, gamma=GAMMA, cov_var=COV, key=99, index=5,
                                  pos0=pos0[:n_ep], debug=True)
        first = {k: out[k][:, : T * E] for k in ("obs", "acts", "log_probs", "rtgs", "eps")}
        first.update(ep_returns=out["ep_returns"][:E], pos=out["pos"][0], final_pos=out["final_pos"][0],
                     final_vel=out["final_vel"][0])
        if base is None:
            base = first
        for k, v in first.items():
            assert torch.equal(v, base[k]), (k, plans[-1])
    print(f"tag_rollout plan invariance {dtype}: plans {plans}")
    if h100_sxm():
        assert {p["rw"] for p in plans} == {1, 4} and len({p["wpb"] for p in plans}) == 5
        if dtype == F64:
            assert {p["stage"] for p in plans} == {0, 1}


def test_environment_keeps_its_own_final_state_when_the_caller_holds_the_buffers():
    """With ``final_pos`` / ``final_vel`` in ``out=``, the environment gets a copy of the last episode's final state:
    the next rollout into the same buffers does not move it."""
    env = tag_env(E=8, dtype=F32)
    actors = actors_for(env, (16,), "own", F32)
    bufs = dict(final_pos=torch.empty(2, 8, env.A, 2, device=DEV), final_vel=torch.empty(2, 8, env.A, 2, device=DEV))
    tag_rollout.rollout(env, actors, T=3, n_ep=2, gamma=GAMMA, cov_var=COV, out=bufs)
    pos, vel = env.pos.clone(), env.vel.clone()
    assert torch.equal(pos, bufs["final_pos"][-1]) and torch.equal(vel, bufs["final_vel"][-1])
    bufs["final_pos"].fill_(float("nan"))
    bufs["final_vel"].fill_(float("nan"))
    assert torch.equal(env.pos, pos) and torch.equal(env.vel, vel)


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible CUDA devices")
def test_actors_and_outputs_on_another_device_are_rejected_before_launch():
    env = tag_env(E=4, dtype=F32)
    actors = actors_for(env, (16,), "own", F32)
    moved = [copy.deepcopy(actors[0]).to("cuda:1")] + actors[1:]
    with pytest.raises(ValueError, match="cuda:1"):
        tag_rollout.rollout(env, moved, T=2, n_ep=1, gamma=GAMMA, cov_var=COV)
    with pytest.raises(ValueError, match="cuda:1"):
        tag_rollout.launch_plan(env, moved, 2, 1)
    bad = dict(rtgs=torch.empty(3, 8, device="cuda:1"))
    with pytest.raises(ValueError, match="out\\['rtgs'\\]"):
        tag_rollout.rollout(env, actors, T=2, n_ep=1, gamma=GAMMA, cov_var=COV, out=bad)
