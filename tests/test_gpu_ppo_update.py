"""The PPO update kernels (ops/csrc/ppo_update.cu) against float64 autograd of ``DistPPOProblem.local_batch_loss`` /
``update_advantage`` at the same parameters and batch, and the trainers that run them.

fp64 kernels: advantages and losses within 1e-12 (relative, per node), every gradient tensor within 1e-9 (the per-step
bound of DESIGN §5).  fp32 kernels: per-tensor error against the fp64 oracle at most 4x that of the torch fp32 CUDA path,
with a floor of a few fp32 ulps of the tensor's norm.

The loss is piecewise smooth: its gradient jumps at every ReLU kink and at both clip edges.  A sample within rounding
distance of a jump takes either branch in any fp32 implementation, and one sample that takes the other branch moves a
gradient summed over R samples by about 1/sqrt(R) (3e-4 at 204,800).  So the recorded batches keep every hidden
pre-activation and every ratio a margin away from the jumps (``_batch``); the yardstick then measures rounding, not
which side of a kink a sample happened to land on.
"""
import networkx as nx
import pytest
import torch

from nn_distributed_training_b200.ops import ppo_update
from nn_distributed_training_b200.rl import DSGDPPO, DSGTPPO, DiNNOPPO, PPO, DistPPOProblem, FFReLUNet, SimpleTagEnv
from ppo_oracle import F32_FLOOR, KINK_MARGIN, make_batch, rel

pytestmark = pytest.mark.gpu
DEV = "cuda"
COV, CLIP = 0.5, 0.2


def _problem(N, hidden, dtype, n_good=1, seed=0, **kw):
    env = SimpleTagEnv(num_envs=2, num_good=n_good, num_adversaries=N, num_obstacles=0, max_cycles=5, device=DEV,
                       dtype=dtype)
    d0 = env.observation_spaces["adversary_0"].shape[0]
    torch.manual_seed(seed)
    graph = nx.wheel_graph(N) if N >= 3 else nx.path_graph(N)
    pr = DistPPOProblem(FFReLUNet([d0, *hidden, 5], dtype=dtype), FFReLUNet([d0, *hidden, 1], dtype=dtype), graph,
                        env, clip=CLIP, **kw)
    for i in range(1, N):   # distinct nodes
        with torch.no_grad():
            for p in pr.models[i].parameters():
                p.add_(0.05 * torch.randn_like(p))
    return pr


def _batch(pr, R, seed=1, spread=0.3, kink_margin=KINK_MARGIN):
    """A recorded batch [N, R, ...] from ``ppo_oracle.make_batch``: acts around the current actor means, so the ratios
    spread around 1 and some clip; no hidden pre-activation within ``kink_margin`` of a ReLU kink."""
    return make_batch([pr.models[i].actor for i in range(pr.N)], [pr.models[i].critic for i in range(pr.N)], R, CLIP,
                      COV, seed=seed, spread=spread, kink_margin=kink_margin)


def _load(pr, batch):
    pr._stack_batch({k: v.to(next(pr.models[0].parameters()).dtype) for k, v in batch.items()})


def _copy_params(dst, src):
    with torch.no_grad():
        for i in range(dst.N):
            for p, q in zip(dst.models[i].parameters(), src.models[i].parameters()):
                p.copy_(q)


def _autograd(pr):
    """Per-node (losses [2], grads) of local_batch_loss under the torch update path."""
    out = []
    for i in range(pr.N):
        a, c = pr.ev_ppo_loss(i)
        g = torch.autograd.grad(a + c, list(pr.models[i].parameters()))
        out.append((torch.stack([a.detach(), c.detach()]), g))
    return out


def _kernel(pr, adv=None):
    grads = [[torch.empty_like(p) for p in pr.models[i].parameters()] for i in range(pr.N)]
    adv = pr._adv if adv is None else adv
    b = pr._batch
    losses = ppo_update.grads(pr.actors, pr.critics, b["obs"], b["acts"], b["log_probs"], b["rtgs"], adv, CLIP, COV, grads)
    return losses, grads


CASES = [   # (N, hidden, n_good, R)
    (3, (64, 64, 64), 1, 800),
    (1, (64, 64, 64), 1, 33),
    (3, (32,), 1, 31),
    (7, (64, 64, 64, 64), 1, 33),
    (3, (64, 64, 64), 2, 1),       # another obs_dim (14)
    (3, (64, 64, 64), 1, 204_800),
]


@pytest.mark.parametrize("N,hidden,n_good,R", CASES)
def test_fp64_against_autograd(N, hidden, n_good, R):
    pr = _problem(N, hidden, torch.float64, n_good=n_good, update_backend="cuda")
    ref = _problem(N, hidden, torch.float64, n_good=n_good)
    _copy_params(ref, pr)
    batch = _batch(pr, R)
    _load(pr, batch)
    _load(ref, batch)
    pr.update_advantage()
    ref.update_advantage()
    for i in range(N):
        if R == 1:   # unbiased std of one sample
            assert torch.isnan(pr.A_k[i]).all() and torch.isnan(ref.A_k[i]).all()
        else:
            assert rel(pr.A_k[i], ref.A_k[i]) < 1e-12
    adv = pr._adv if R > 1 else torch.randn(N, R, device=DEV, dtype=torch.float64)
    if R == 1:
        ref.A_k = {i: adv[i] for i in range(N)}
    losses, grads = _kernel(pr, adv)
    for i, (l_ref, g_ref) in enumerate(_autograd(ref)):
        assert rel(losses[i], l_ref) < 1e-12, (i, losses[i], l_ref)
        for k, (g, gr) in enumerate(zip(grads[i], g_ref)):
            assert rel(g, gr) < 1e-9, (i, k, rel(g, gr))


@pytest.mark.parametrize("N,hidden,n_good,R", [c for c in CASES if c[3] > 1])
def test_fp32_against_the_torch_fp32_yardstick(N, hidden, n_good, R):
    ref = _problem(N, hidden, torch.float64, n_good=n_good)
    t32 = _problem(N, hidden, torch.float32, n_good=n_good)
    k32 = _problem(N, hidden, torch.float32, n_good=n_good, update_backend="cuda")
    _copy_params(t32, ref)
    _copy_params(k32, ref)
    batch = {k: v.float() for k, v in _batch(ref, R).items()}   # fp32-representable batch for all three
    for pr in (ref, t32, k32):
        _load(pr, batch)
        pr.update_advantage()
    for i in range(N):
        e_t, e_k = rel(t32.A_k[i], ref.A_k[i]), rel(k32.A_k[i], ref.A_k[i])
        assert e_k <= 4 * max(e_t, F32_FLOOR), ("adv", i, e_k, e_t)
    adv = k32._adv.double()   # one advantage for all three, so the gradients compare the update alone
    ref.A_k = {i: adv[i] for i in range(N)}
    t32.A_k = {i: adv[i].float() for i in range(N)}
    losses, grads = _kernel(k32, adv.float())
    for i, ((l_ref, g_ref), (l_t, g_t)) in enumerate(zip(_autograd(ref), _autograd(t32))):
        for n in range(2):
            e_t, e_k = rel(l_t[n], l_ref[n]), rel(losses[i, n], l_ref[n])
            assert e_k <= 4 * max(e_t, F32_FLOOR), ("loss", i, n, e_k, e_t)
        for k, (g, gt, gr) in enumerate(zip(grads[i], g_t, g_ref)):
            e_t, e_k = rel(gt, gr), rel(g, gr)
            assert e_k <= 4 * max(e_t, F32_FLOOR), ("grad", i, k, e_k, e_t)


def test_clip_semantics_against_autograd():
    """Ratios 0.5, 0.79, 1.0, 1.21, 2.0 under positive, negative and zero advantages."""
    pr = _problem(3, (64, 64, 64), torch.float64, update_backend="cuda")
    ref = _problem(3, (64, 64, 64), torch.float64)
    _copy_params(ref, pr)
    R = 15
    batch = _batch(pr, R)
    ratios = torch.tensor([0.5, 0.79, 1.0, 1.21, 2.0], device=DEV, dtype=torch.float64).repeat(3)
    advs = torch.tensor([1.0, -1.0, 0.0], device=DEV, dtype=torch.float64).repeat_interleave(5)
    with torch.no_grad():
        mean = torch.stack([pr.models[i].actor(batch["obs"][i]) for i in range(3)])
    batch["log_probs"] = pr._log_prob(mean, batch["acts"]) - torch.log(ratios)
    _load(pr, batch)
    _load(ref, batch)
    adv = torch.stack([advs * (1 + 0.1 * i) for i in range(3)])
    ref.A_k = {i: adv[i] for i in range(3)}
    losses, grads = _kernel(pr, adv)
    for i, (l_ref, g_ref) in enumerate(_autograd(ref)):
        assert rel(losses[i], l_ref) < 1e-12
        for g, gr in zip(grads[i], g_ref):
            assert rel(g, gr) < 1e-12


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_bitwise_determinism_and_arena_padding(dtype):
    from nn_distributed_training_b200.optimizers.base import ReferenceProblemAdapter
    pr = _problem(3, (64, 64, 64), dtype, update_backend="cuda")
    ad = ReferenceProblemAdapter(pr, DEV)
    _load(pr, _batch(pr, 4096))
    pr.update_advantage()
    adv1 = pr._adv.clone()
    pr.update_advantage()
    assert torch.equal(adv1, pr._adv)
    ad.arena.grad.fill_(0)
    l1 = ad.compute_grads().clone()
    g1 = ad.arena.grad.clone()
    ad.compute_grads()
    assert torch.equal(l1, ad.last_losses) and torch.equal(g1, ad.arena.grad)
    mask = torch.ones(ad.arena.n_pad, dtype=torch.bool, device=DEV)
    for s in ad.layout.slots:
        mask[s.offset: s.offset + s.numel] = False
    assert mask.any() and (g1[:, mask] == 0).all()          # alignment holes stay zero
    assert torch.isfinite(g1).all() and (g1[:, ~mask] != 0).any()


TRAINERS = [
    (DiNNOPPO, {"rho_init": 1.0, "rho_scaling": 1.0, "primal_lr_start": 3e-4, "primal_lr_finish": 1e-3,
                "lr_decay_type": "constant", "persistant_primal_opt": False, "primal_iterations": 5,
                "outer_iterations": 10 ** 6}),
    (DSGDPPO, {"alpha0": 3e-3, "mu": 0.0}),
    (DSGTPPO, {"alpha_actor": 3e-3, "alpha_critic": 1e-2, "init_grads": True}),
    (DSGTPPO, {"alpha": 3e-3, "mixing_order": "reference"}),   # per-node autograd through the A_k views
]


@pytest.mark.parametrize("cls,conf", TRAINERS)
def test_whole_runs_match_the_torch_update(cls, conf):
    """3 rounds x 5 primal steps on one fixed recorded batch, fp64: cuda and torch update paths end within 1e-8."""
    out = []
    for backend in ("torch", "cuda"):
        pr = _problem(3, (64, 64, 64), torch.float64, update_backend=backend, n_updates_per_iteration=5)
        batch = _batch(pr, 800)
        tr = cls(pr, DEV, dict(conf, max_rl_timesteps=10 ** 9, writeout=False))
        start = torch.cat([torch.nn.utils.parameters_to_vector(pr.models[i].parameters()) for i in range(3)])
        for k in range(3):
            _load(pr, batch)
            pr.update_advantage()
            if k == 0:
                tr.inner._before_training()   # DSGT's init_grads
            tr._consensus(k)
            pr.check_update()
        out.append(torch.cat([torch.nn.utils.parameters_to_vector(pr.models[i].parameters()) for i in range(3)]))
        assert not torch.equal(out[-1], start)
    assert rel(out[1], out[0]) < 1e-8


def test_end_to_end_dinno_ppo_with_both_kernels(tmp_path):
    from nn_distributed_training_b200.rl.train_common import common_conf, make_problem, parse_args
    args = parse_args(["--num_envs", "16", "--device", "cuda", "--rollout", "cuda", "--update", "cuda", "--seed", "0",
                       "--max_rl_timesteps", "6000", "--out_dir", str(tmp_path), "--no_writeout"])
    pr, hyper = make_problem(args)
    assert pr.update_backend == "cuda"
    conf = dict(common_conf(args), rho_init=1.0, rho_scaling=1.0, primal_lr_start=hyper["lr"], primal_lr_finish=0.001,
                lr_decay_type="constant", persistant_primal_opt=False, primal_iterations=5, outer_iterations=10 ** 6)
    before = torch.nn.utils.parameters_to_vector(pr.models[0].parameters()).clone()
    tr = DiNNOPPO(pr, DEV, conf)
    tr.train()
    after = torch.nn.utils.parameters_to_vector(pr.models[0].parameters())
    assert len(tr.avg_ep_rews) >= 2 and torch.isfinite(after).all() and not torch.equal(before, after)


def test_end_to_end_ppo_learn():
    env = SimpleTagEnv(num_envs=16, num_good=1, num_adversaries=3, num_obstacles=8, max_cycles=50, device=DEV)
    m = PPO(FFReLUNet, env, timesteps_per_batch=2000, max_timesteps_per_episode=200, rollout_backend="cuda",
            update_backend="cuda", lr=3e-4, save_freq=10 ** 6, seed=0)
    before = torch.nn.utils.parameters_to_vector(m.actor.parameters()).clone()
    m.learn(total_timesteps=6000)
    after = torch.nn.utils.parameters_to_vector(m.actor.parameters())
    assert len(m.avg_ep_rews) >= 2 and torch.isfinite(after).all() and not torch.equal(before, after)


def test_nan_actor_raises_by_the_end_of_the_iteration():
    pr = _problem(3, (64, 64, 64), torch.float32, update_backend="cuda", n_updates_per_iteration=2)
    with torch.no_grad():
        pr.models[1].actor.seq[0].weight[0, 0] = float("nan")
    tr = DSGDPPO(pr, DEV, {"alpha0": 1e-3, "mu": 0.0, "max_rl_timesteps": 10 ** 9, "writeout": False})
    _load(pr, _batch(pr, 64))
    pr.update_advantage()
    tr._consensus(0)
    with pytest.raises(NameError, match="actor returning something weird"):
        pr.check_update()


def test_nan_actor_raises_from_the_next_advantage_pass_without_a_check():
    """A driver that never calls check_update() still hears of it before the next iteration's update."""
    pr = _problem(3, (64, 64, 64), torch.float32, update_backend="cuda", n_updates_per_iteration=2)
    with torch.no_grad():
        pr.models[0].actor.seq[2].bias[3] = float("inf")
    tr = DSGDPPO(pr, DEV, {"alpha0": 1e-3, "mu": 0.0, "max_rl_timesteps": 10 ** 9, "writeout": False})
    batch = _batch(pr, 64, kink_margin=0.0)
    _load(pr, batch)
    pr.update_advantage()
    tr._consensus(0)
    _load(pr, batch)
    with pytest.raises(NameError, match="actor returning something weird"):
        pr.update_advantage()
