"""The PPO update kernels (ops/csrc/ppo_update.cu) at every instantiation, launch plan and shape edge, against the
float64 oracle of tests/ppo_oracle.py.

``ppo_update.grads`` / ``advantages`` run directly on per-node ``FFReLUNet`` pairs: 1, 2 and 8 nodes; no hidden
layer (no backward propagation), width-1, 15- and 17-wide layers (padding to 16 and 32), ``(1, 7, 64)`` and four
layers of 64; obs widths 1, 8, 33 and 64; actors and critics of different depth and width; R in {1, 2, tm - 1, tm,
tm + 1, 257}, an R whose trailing chunks are empty (chosen from ``ppo_update.launch_plan``) and an advantage pass over
millions of rows.  fp64: losses and advantages within 1e-12, gradients within 1e-9 (relative).  fp32: at most 4x the
error of torch fp32 (the larger of two row orders), with a floor of a few fp32 ulps of the summed terms' size.  Every
output is poisoned with NaN before each launch and sits between guard values in a larger buffer; two launches must be
bitwise equal.
"""
import copy

import pytest
import torch

from nn_distributed_training_b200.ops import ppo_update
from nn_distributed_training_b200.rl import FFReLUNet
from kernel_oracles import Guarded, fp32_references
from ppo_oracle import (advantages_reference, check_adv, check_losses_and_grads, gradient_scales, make_batch,
                        ppo_reference)

pytestmark = pytest.mark.gpu
DEV = "cuda"
COV, CLIP = 0.5, 0.2
DTYPES = [torch.float64, torch.float32]
DT_ID = {torch.float64: "fp64", torch.float32: "fp32"}

SHAPES = {   # name: (N, obs width, actor hidden layers, critic hidden layers)
    "no-hidden": (1, 8, (), ()),
    "width-1": (2, 1, (1,), (1,)),
    "pad-15-17": (8, 33, (15,), (17,)),
    "deep-mixed": (2, 64, (1, 7, 64), (64,)),
    "four-64": (1, 64, (64,) * 4, (64,) * 4),       # fp64: 32-row tiles exceed the opt-in shared memory
    "unequal-n8": (8, 12, (64,) * 4, (32,)),
}


def _nets(name, dtype, seed=0):
    N, d0, ah, ch = SHAPES[name]
    torch.manual_seed(seed)
    actors = [FFReLUNet([d0, *ah, 5], dtype=dtype).to(DEV) for _ in range(N)]
    critics = [FFReLUNet([d0, *ch, 1], dtype=dtype).to(DEV) for _ in range(N)]
    return actors, critics


def _per(R, plan):
    tm, chunks = plan["tm"], plan["chunks"]
    return -(-(-(-R // chunks)) // tm) * tm


def _has_empty_chunk(R, plan):
    return plan["chunks"] * _per(R, plan) - R >= _per(R, plan)


def r_with_empty_chunks(actors, critics):
    """The smallest R = k tm + 1 whose plan leaves the trailing chunks without rows."""
    tm = ppo_update.launch_plan(actors, critics, 1)["tm"]
    for k in range(1, 4096):
        R = k * tm + 1
        if _has_empty_chunk(R, ppo_update.launch_plan(actors, critics, R)):
            return R
    raise AssertionError("no R up to 4096 tiles leaves a chunk empty")


def sizes(actors, critics):
    tm = ppo_update.launch_plan(actors, critics, 1)["tm"]
    return sorted({1, 2, tm - 1, tm, tm + 1, 257, r_with_empty_chunks(actors, critics)})


def run_grads(actors, critics, b, adv):
    """One ``grads`` launch into poisoned, guarded gradient and loss buffers, with a workspace whose partial-sum
    slots all hold NaN (bytes 0xFF): a CTA that skipped its slot, such as an empty trailing chunk's, shows as NaN."""
    N, R = adv.shape
    dt = adv.dtype
    shapes = [p.shape for i in range(N) for p in (*actors[i].parameters(), *critics[i].parameters())]
    gbuf, lbuf = Guarded(shapes, dt, DEV), Guarded([(N, 2)], dt, DEV)
    per_node = len(shapes) // N
    grads = [gbuf.views[i * per_node: (i + 1) * per_node] for i in range(N)]
    nonfinite = torch.zeros(1, dtype=torch.int32, device=DEV)
    nw = ppo_update.launch_plan(actors, critics, R)["work_bytes"]
    work = torch.full((nw + 64,), 0xFF, dtype=torch.uint8, device=DEV)
    ppo_update.grads(actors, critics, b["obs"], b["acts"], b["log_probs"], b["rtgs"], adv, CLIP, COV, grads,
                     nonfinite=nonfinite, losses_out=lbuf.views[0], workspace=work)
    torch.cuda.synchronize()
    gbuf.assert_guards("gradients")
    lbuf.assert_guards("losses")
    assert (work[nw:] == 0xFF).all(), "a write past the workspace"
    assert nonfinite.item() == 0
    return lbuf.views[0].clone(), [[g.clone() for g in node] for node in grads]


def run_advantages(critics, b):
    N, R = b["rtgs"].shape
    out = Guarded([(N, R)], b["rtgs"].dtype, DEV)
    ppo_update.advantages(critics, b["obs"], b["rtgs"], out=out.views[0])
    torch.cuda.synchronize()
    out.assert_guards("advantages")
    return out.views[0].clone()


def _bitwise(a, b):
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("name", list(SHAPES))
def test_grads_and_advantages_against_the_oracle(name, dtype):
    actors, critics = _nets(name, dtype)
    N = len(actors)
    worst, plans = 0.0, set()
    with fp32_references():
        for R in sizes(actors, critics):
            what = (name, DT_ID[dtype], R)
            plans.add(tuple(ppo_update.launch_plan(actors, critics, R).values()))
            b = make_batch(actors, critics, R, CLIP, COV, seed=R)
            adv = run_advantages(critics, b)
            assert _bitwise(adv, run_advantages(critics, b)), (what, "advantages differ between launches")
            for i in range(N):
                if R == 1:   # the unbiased std of one sample
                    assert adv[i].isnan().all(), what
                    continue
                ref = advantages_reference(critics[i], b["obs"][i], b["rtgs"][i])
                t32 = advantages_reference(critics[i], b["obs"][i], b["rtgs"][i], dtype=torch.float32)
                worst = max(worst, check_adv(dtype, adv[i], ref, t32, what + (i, "adv")))
            if R == 1:
                adv = torch.randn(N, R, device=DEV, dtype=dtype)
            losses, grads = run_grads(actors, critics, b, adv)
            l2, g2 = run_grads(actors, critics, b, adv)
            same = torch.equal(losses, l2) and all(torch.equal(x, y) for gi, hi in zip(grads, g2)
                                                   for x, y in zip(gi, hi))
            assert same, (what, "gradients differ between launches")
            for i in range(N):
                row = [b[k][i] for k in ("obs", "acts", "log_probs", "rtgs")] + [adv[i]]
                ref = ppo_reference(actors[i], critics[i], *row, CLIP, COV)
                t32 = [ppo_reference(actors[i], critics[i], *rows, CLIP, COV, dtype=torch.float32)   # two row orders
                       for rows in (row, [t.flip(0) for t in row])] if dtype == torch.float32 else ()
                gs = gradient_scales(actors[i], critics[i], *row, CLIP, COV) if dtype == torch.float32 else None
                worst = max(worst, check_losses_and_grads(dtype, losses[i], grads[i], ref, t32, what + (i,), gs))
    kind = "error / bound" if dtype == torch.float64 else "error / torch fp32 error"
    print(f"ppo_update {name} {DT_ID[dtype]}: plans (tm, chunks, smem) {sorted(plans)}; worst {kind} {worst:.3g}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_advantages_over_millions_of_rows(dtype):
    """adv_norm_kernel's strided sums and block tree over 3,000,017 rows per node (not a multiple of 256)."""
    actors, critics = _nets("pad-15-17", dtype)
    critics = critics[:2]
    b = make_batch(None, critics, 3_000_017, CLIP, COV)
    adv = run_advantages(critics, b)
    with fp32_references():
        worst = 0.0
        for i in range(2):
            ref = advantages_reference(critics[i], b["obs"][i], b["rtgs"][i])
            t32 = advantages_reference(critics[i], b["obs"][i], b["rtgs"][i], dtype=torch.float32)
            worst = max(worst, check_adv(dtype, adv[i], ref, t32, ("millions", DT_ID[dtype], i)))
    print(f"ppo_update advantages R=3,000,017 {DT_ID[dtype]}: worst {worst:.3g}")


def test_plan_coverage():
    """The cases above reach 16- and 32-row tiles, one chunk, several chunks with an empty trailing one, and N = 8."""
    props = torch.cuda.get_device_properties(0)
    if props.shared_memory_per_block_optin != 227 * 1024:
        pytest.skip(f"the tile choices are those of 227 KB of opt-in shared memory; this device has "
                    f"{props.shared_memory_per_block_optin} B")
    seen = dict(tm16=False, tm32=False, one_chunk=False, empty_chunk=False, n8=False)
    for name in SHAPES:
        for dtype in DTYPES:
            actors, critics = _nets(name, dtype)
            for R in sizes(actors, critics):
                p = ppo_update.launch_plan(actors, critics, R)
                seen[f"tm{p['tm']}"] = True
                seen["one_chunk"] |= p["chunks"] == 1
                seen["empty_chunk"] |= p["chunks"] > 1 and _has_empty_chunk(R, p)
                seen["n8"] |= len(actors) == 8
    assert all(seen.values()), seen
    four = _nets("four-64", torch.float64)
    assert ppo_update.launch_plan(*four, 1000)["tm"] == 16


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible CUDA devices")
def test_networks_and_outputs_on_another_device_are_rejected_before_launch():
    actors, critics = _nets("pad-15-17", torch.float64)
    b = make_batch(actors, critics, 40, CLIP, COV)
    adv = run_advantages(critics, b)
    other = [FFReLUNet([33, 15, 5], dtype=torch.float64).to("cuda:1")] + actors[1:]
    grads = [[torch.empty_like(p) for p in (*actors[i].parameters(), *critics[i].parameters())] for i in range(8)]
    args = (b["obs"], b["acts"], b["log_probs"], b["rtgs"], adv, CLIP, COV)
    with pytest.raises(ValueError, match="cuda:1"):
        ppo_update.grads(other, critics, *args, grads)
    with pytest.raises(ValueError, match="cuda:1"):
        ppo_update.advantages([copy.deepcopy(critics[0]).to("cuda:1")] + critics[1:], b["obs"], b["rtgs"])
    on1 = dict(dtype=torch.float64, device="cuda:1")
    with pytest.raises(ValueError, match="out: .* on cuda:1"):
        ppo_update.advantages(critics, b["obs"], b["rtgs"], out=torch.empty(8, 40, **on1))
    with pytest.raises(ValueError, match="losses_out: .* on cuda:1"):
        ppo_update.grads(actors, critics, *args, grads, losses_out=torch.empty(8, 2, **on1))
    with pytest.raises(ValueError, match="workspace: .* on cuda:1"):
        ppo_update.grads(actors, critics, *args, grads,
                         workspace=torch.empty(1 << 20, dtype=torch.uint8, device="cuda:1"))
    grads[3][2] = grads[3][2].to("cuda:1")
    with pytest.raises(ValueError, match="grad_out.* on cuda:1"):
        ppo_update.grads(actors, critics, *args, grads)
