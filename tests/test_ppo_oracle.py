"""CPU checks of the PPO update's float64 oracle (tests/ppo_oracle.py): it is the torch update path's math, and the
comparisons the GPU tests make reject the defects a tiled, chunked kernel could make."""
import networkx as nx
import pytest
import torch

from nn_distributed_training_b200.rl import DistPPOProblem, FFReLUNet, SimpleTagEnv
from ppo_oracle import (advantages_reference, check_adv, check_fp32, check_fp64, check_losses_and_grads,
                        gradient_scales, log_prob, make_batch, mlp, ppo_reference, weights)

COV, CLIP = 0.5, 0.2


def test_oracle_is_the_torch_update_path():
    """``ppo_reference`` / ``advantages_reference`` equal ``DistPPOProblem.ev_ppo_loss`` under autograd and
    ``update_advantage`` (torch update path, float64) to rounding."""
    env = SimpleTagEnv(num_envs=2, num_good=1, num_adversaries=3, num_obstacles=0, max_cycles=5, dtype=torch.float64)
    torch.manual_seed(0)
    pr = DistPPOProblem(FFReLUNet([12, 17, 5], dtype=torch.float64), FFReLUNet([12, 15, 15, 1], dtype=torch.float64),
                        nx.wheel_graph(3), env, clip=CLIP)
    with torch.no_grad():
        for i in range(1, 3):
            for p in pr.models[i].parameters():
                p.add_(0.05 * torch.randn_like(p))
    actors, critics = [pr.models[i].actor for i in range(3)], [pr.models[i].critic for i in range(3)]
    b = make_batch(actors, critics, 300, CLIP, pr.cov_var)
    pr._stack_batch(b)
    pr.update_advantage()
    for i in range(3):
        adv = advantages_reference(critics[i], b["obs"][i], b["rtgs"][i])
        assert (adv - pr.A_k[i]).norm() <= 1e-13 * adv.norm()
        a, c = pr.ev_ppo_loss(i)
        g = torch.autograd.grad(a + c, list(pr.models[i].parameters()))
        losses, grads, _ = ppo_reference(actors[i], critics[i], b["obs"][i], b["acts"][i], b["log_probs"][i],
                                      b["rtgs"][i], pr.A_k[i], CLIP, pr.cov_var)
        assert (losses - torch.stack([a, c]).detach()).abs().max() <= 1e-13 * losses.abs().max()
        assert len(grads) == len(g)
        for x, y in zip(grads, g):
            assert x.shape == y.shape and (x - y).norm() <= 1e-13 * y.norm()


# ---- planted defects -------------------------------------------------------------------------------------------------
R = 100   # three 32-row tiles and a partial one of 4 rows; with chunks of 64 rows, a second chunk of 36


@pytest.fixture(scope="module")
def node():
    """One fp32 node (fp32-representable parameters and batch), its float64 oracle and its torch fp32 yardstick."""
    torch.manual_seed(3)
    actor, critic = FFReLUNet([12, 15, 5], dtype=torch.float32), FFReLUNet([12, 17, 1], dtype=torch.float32)
    b = {k: v[0] for k, v in make_batch([actor], [critic], R, CLIP, COV).items()}
    adv = advantages_reference(critic, b["obs"], b["rtgs"]).float()
    args = (actor, critic, b["obs"], b["acts"], b["log_probs"], b["rtgs"], adv, CLIP, COV)
    return dict(args=args, ref=ppo_reference(*args), t32=ppo_reference(*args, dtype=torch.float32), batch=b)


def _flat(out):
    losses, grads = out[:2]
    return [losses[0], losses[1], *grads]


def _rows(*spans):
    w = torch.ones(R, dtype=torch.float64)
    for lo, hi, v in spans:
        w[lo:hi] = v
    return w


DEFECTS = {
    "a 32-row tile dropped": lambda n: ppo_reference(*n["args"], row_weight=_rows((32, 64, 0.0))),
    "the second 64-row chunk's partial dropped": lambda n: ppo_reference(*n["args"], row_weight=_rows((64, R, 0.0))),
    "the last partial tile counted twice": lambda n: ppo_reference(*n["args"], row_weight=_rows((96, R, 2.0))),
    "a padded column leaking into a bias gradient": lambda n: _leak(n["ref"]),
}


def _leak(ref):
    """Layer 0's 15 outputs sit in a 16-wide tile: the gradient sum of column 0 lands in bias entry 14 as well."""
    losses, grads, scales = ref
    grads = [g.clone() for g in grads]
    grads[1][14] += grads[1][0]
    return losses, grads, scales


def test_comparisons_accept_the_oracle_and_torch_fp32(node):
    check_fp64(*node["ref"][:2], *node["ref"])
    check_fp32(_flat(node["t32"]), _flat(node["ref"]), _flat(node["t32"]))


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_comparisons_reject_planted_defects(node, defect):
    bad = DEFECTS[defect](node)
    with pytest.raises(AssertionError):
        check_fp64(*bad[:2], *node["ref"])
    with pytest.raises(AssertionError):
        check_fp32(_flat(bad), _flat(node["ref"]), _flat(node["t32"]))


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_the_gpu_tests_fp32_comparison_rejects_planted_defects(node, defect):
    """The comparison the fp32 GPU test makes (``check_losses_and_grads`` with ``gradient_scales`` floors and two torch
    fp32 row orders) accepts torch fp32 and still rejects every defect."""
    args = node["args"]
    rows = list(args[2:7])
    flipped = ppo_reference(*args[:2], *[t.flip(0) for t in rows], CLIP, COV, dtype=torch.float32)
    t32 = [node["t32"], flipped]
    gs = gradient_scales(*args)
    assert check_losses_and_grads(torch.float32, *node["t32"][:2], node["ref"], t32, grad_scales=gs) <= 1
    bad = DEFECTS[defect](node)
    with pytest.raises(AssertionError):
        check_losses_and_grads(torch.float32, *bad[:2], node["ref"], t32, grad_scales=gs)


def test_comparisons_reject_the_biased_std(node):
    b, critic = node["batch"], node["args"][1]
    ref = advantages_reference(critic, b["obs"], b["rtgs"])
    t32 = advantages_reference(critic, b["obs"], b["rtgs"], dtype=torch.float32)
    biased = advantages_reference(critic, b["obs"], b["rtgs"], unbiased=False)
    check_adv(torch.float64, ref, ref)
    check_adv(torch.float32, t32, ref, t32)
    with pytest.raises(AssertionError):
        check_adv(torch.float64, biased, ref)
    with pytest.raises(AssertionError):
        check_adv(torch.float32, biased, ref, t32)


def test_comparison_rejects_the_gradient_on_the_open_clip_interval(node):
    """A row whose float64 ratio is exactly 1 - clip or 1 + clip (the clip chosen from that row's ratio, so the edge is
    hit exactly): autograd's clamp passes the gradient there (closed interval), and the kernel must too.  In fp32 such
    a row's ratio lands on either side of the edge, so only the fp64 check can tell; the fp32 batches keep every ratio
    away from the edges instead."""
    actor, critic, obs, acts, old_lp, rtgs, adv, _, cov = node["args"]
    with torch.no_grad():
        ratio = torch.exp(log_prob(mlp(weights(actor), obs.double()), acts.double(), cov) - old_lp.double())
    for side in (-1, 1):
        r = int(torch.nonzero((side * (ratio - 1) > 0.05) & (side * (ratio - 1) < 0.5))[0])
        clip = side * (float(ratio[r]) - 1)                  # exact: 1 -+ clip is ratio[r] again
        assert 1 + side * clip == float(ratio[r])
        args = (actor, critic, obs, acts, old_lp, rtgs, adv, clip, cov)
        ref = ppo_reference(*args)
        check_fp64(*ref[:2], *ref)
        with pytest.raises(AssertionError):
            check_fp64(*ppo_reference(*args, open_clip=True)[:2], *ref)
