"""GPU numerics of the tensor-core MLP kernels vs fp32 PyTorch."""
import copy

import networkx as nx
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.models import FourierNet
from nn_distributed_training_b200.parallel.arena import FlatLayout, NodeArena

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _fp32_references():
    """The fp32 autograd comparisons in this module mean fp32, not TF32."""
    with ko.fp32_references():
        yield


def _arena(shape, scale, L, seed=0):
    torch.manual_seed(seed)
    models = []
    base = FourierNet(shape, scale=scale)
    arena = NodeArena(FlatLayout.from_module(base), L, DEV, torch.float32)
    for l in range(L):
        m = FourierNet(shape, scale=scale).to(DEV)
        arena.attach(l, m)
        models.append(m)
    return arena, models, base.spec


@pytest.mark.parametrize("h1", [256, 64, 128])
@pytest.mark.parametrize("M", [1000, 128, 77])
def test_mlp_forward_matches_torch(h1, M):
    from nn_distributed_training_b200.ops.mlp_fused import MlpForward
    arena, models, spec = _arena([2, h1, 64, 64, 64, 1], 0.05, 3)
    x = (torch.rand(M, 2, device=DEV) - 0.5) * 1500
    out = MlpForward(arena, spec, 3, torch.device(DEV))(x)
    torch.cuda.synchronize()
    for l, m in enumerate(models):
        with torch.no_grad():
            ref = m(x).reshape(-1)
        # bf16 operands, fp32 accumulation
        assert (out[l] - ref).abs().max().item() < 2e-2, (out[l] - ref).abs().max().item()
        assert (out[l] - ref).abs().mean().item() < 3e-3


def _density_problem(backend, h1=256, B=1000, M=3000, N=3, loss="BCE", seed=0):
    import networkx as nx
    from nn_distributed_training_b200.data.shards import Shard
    from nn_distributed_training_b200.problems import DistDensityProblem
    g = torch.Generator().manual_seed(seed)
    shards = []
    for i in range(N):
        x = (torch.rand(M, 2, generator=g) - 0.5) * 1200
        y = (torch.rand(M, generator=g) < 0.3).float()
        shards.append(Shard(x, y))
    val = Shard((torch.rand(500, 2, generator=g) - 0.5) * 1200, (torch.rand(500, generator=g) < 0.3).float())
    conf = {"problem_name": "d", "train_batch_size": B, "val_batch_size": 200,
            "metrics": ["forward_pass_count", "validation_loss", "consensus_error", "current_epoch"],
            "metrics_config": {"evaluate_frequency": 100}, "optimizer_config": {}}
    torch.manual_seed(seed)
    base = FourierNet([2, h1, 64, 64, 64, 1], scale=0.05)
    lossf = {"BCE": torch.nn.BCELoss(), "MSE": torch.nn.MSELoss(), "L1": torch.nn.L1Loss()}[loss]
    return DistDensityProblem(nx.cycle_graph(N), base, lossf, shards, val, DEV, conf, backend=backend, seed=3)


@pytest.mark.parametrize("h1,B,loss", [(256, 1000, "BCE"), (256, 128, "BCE"), (64, 300, "MSE"), (128, 1500, "L1"), (256, 2048, "BCE")])
def test_mlp_train_kernel_matches_autograd(h1, B, loss):
    """Tolerances: the kernel feeds bf16 operands to the tensor cores (fp32 accumulation) and is compared with fp32 autograd, so per-tensor
    gradient errors are a few percent and grow towards the first layer (three bf16 roundings of dH on the way back).  That this is
    harmless for training is a question for an end-to-end run (dist_online_dense_PAPER on the reference's real floor plan
    against the fp64 reference), not for this test."""
    fused = _density_problem("fused", h1=h1, B=B, loss=loss)
    ref = _density_problem("torch", h1=h1, B=B, loss=loss)
    assert fused.backend == "fused" and ref.backend == "torch"
    ref.arena.theta.copy_(fused.arena.theta)
    for step in range(4):
        lf = fused.compute_grads().clone()
        lr = ref.compute_grads().clone()
        torch.testing.assert_close(lf, lr, rtol=3e-2, atol=3e-3)
        for s in fused.layout.slots:
            a = fused.arena.grad[:, s.offset: s.offset + s.numel]
            b = ref.arena.grad[:, s.offset: s.offset + s.numel]
            rel = ((a - b).norm() / b.norm().clamp_min(1e-9)).item()
            assert rel < (0.12 if s.name.startswith('seq.0') else 6e-2), (s.name, rel, step)  # bf16 rounding accumulates towards layer 1
    assert (fused.calls == ref.calls).all()


def test_mlp_eval_matches_torch():
    fused = _density_problem("fused")
    ref = _density_problem("torch")
    ref.arena.theta.copy_(fused.arena.theta)
    torch.testing.assert_close(fused._val_losses_local(), ref._val_losses_local(), rtol=2e-2, atol=2e-2)


def _online_problem(backend, tmp, opt_conf, B=700):
    import glob, os
    import numpy as np
    from nn_distributed_training_b200.floorplans.lidar import Lidar2D, OnlineTrajectoryLidarDataset, RandomPoseLidarDataset
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    from nn_distributed_training_b200.problems import DistOnlineDensityProblem
    if not os.path.exists(os.path.join(tmp, "floor_img.png")):
        write_dataset(tmp, n_paths=3, seed=0)
    lidar = Lidar2D(os.path.join(tmp, "floor_img.png"), 8, 0.2, 10, 1.0, 20, 3, border_width=8)
    paths = sorted(glob.glob(os.path.join(tmp, "tight_paths", "*.npy")))
    np.random.seed(0)
    train = [OnlineTrajectoryLidarDataset(lidar, np.load(p), 4, 12, seed=5, node=i) for i, p in enumerate(paths)]
    val = RandomPoseLidarDataset(lidar, 10)
    conf = {"problem_name": "o", "train_batch_size": B, "val_batch_size": 300, "comm_radius": 300.0,
            "dynamic_graph": True, "save_models": False,
            "metrics": ["forward_pass_count", "train_loss_moving_average", "validation_loss", "consensus_error", "current_epoch"],
            "metrics_config": {"evaluate_frequency": 4, "tloss_decay": 0.2, "mesh_only_at_end": True},
            "optimizer_config": opt_conf}
    torch.manual_seed(0)
    base = FourierNet([2, 256, 64, 64, 64, 1], scale=0.05)
    return DistOnlineDensityProblem(base, torch.nn.BCELoss(), train, val, DEV, conf, backend=backend, seed=5)


def test_online_window_sampler_matches_python(tmp_path):
    """The in-kernel sliding-window sampler must draw the rows the Python schedule draws:
    per-step losses of the fused and the autograd path agree across several window switches."""
    oc = {"alg_name": "dsgd", "alpha0": 0.001, "mu": 0.001, "outer_iterations": 2, "profile": False}
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    assert fused.backend == "fused"
    ref.arena.theta.copy_(fused.arena.theta)
    for step in range(12):          # windows hold 12 scans x 80 points = 960 draws: a switch every ~1.4 steps
        lf = fused.compute_grads().clone()
        lr = ref.compute_grads().clone()
        torch.testing.assert_close(lf, lr, rtol=2e-2, atol=2e-3)
    assert (fused.positions() == ref.positions()).all()


def test_online_density_fused_training_tracks_torch_path(tmp_path):
    from nn_distributed_training_b200.optimizers import DiNNO
    oc = {"alg_name": "dinno", "rho_init": 0.3, "rho_scaling": 1.0004, "outer_iterations": 9, "primal_iterations": 3,
          "primal_optimizer": "adam", "persistant_primal_opt": False, "primal_lr_start": 0.001,
          "primal_lr_finish": 0.0001, "lr_decay_type": "log", "profile": False}
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    ref.arena.theta.copy_(fused.arena.theta)
    DiNNO(fused, DEV, oc).train()
    DiNNO(ref, DEV, dict(oc, consensus_backend="torch")).train()
    vf, vr = fused.metrics["validation_loss"][-1], ref.metrics["validation_loss"][-1]
    assert len(fused.metrics["validation_loss"]) == len(ref.metrics["validation_loss"]) == 3
    torch.testing.assert_close(vf, vr, rtol=5e-2, atol=5e-2)
    tf, tr = fused.metrics["train_loss_moving_average"][-1], ref.metrics["train_loss_moving_average"][-1]
    torch.testing.assert_close(tf, tr, rtol=5e-2, atol=2e-2)
    assert fused.forward_cnt == ref.forward_cnt


# ---- generic CUDA-core MLP kernels (csrc/mlp_generic.cu): any widths <= 256, ReLU / Tanh / Sigmoid, fp32 / fp64 ---------
@pytest.mark.parametrize("cls_name,shape,dtype,M", [
    ("FFReLUNet", [12, 64, 64, 64, 5], torch.float32, 2400),        # RL actor (reference RL/dist_rl/model.py)
    ("FFReLUNet", [12, 64, 64, 64, 1], torch.float32, 777),         # RL critic, ragged last tile
    ("FFTanhNet", [2, 37, 129, 3], torch.float64, 100),
    ("FFSigmoidNet", [7, 256, 16, 8], torch.float32, 65),
    ("FFReLUNet", [2, 200, 1], torch.float64, 33),
])
def test_generic_mlp_kernels_match_autograd(cls_name, shape, dtype, M, monkeypatch):
    from nn_distributed_training_b200.models import relu_nn
    torch.manual_seed(0)
    net = getattr(relu_nn, cls_name)(shape, dtype=dtype).to(DEV)
    x = torch.randn(M, shape[0], dtype=dtype, device=DEV, requires_grad=True)
    w = torch.randn(M, shape[-1], dtype=dtype, device=DEV)
    out = net(x)                                   # fused: ops/mlp_generic.py
    (out * w).sum().backward()
    g_fused = [p.grad.clone() for p in net.parameters()]
    gx_fused = x.grad.clone()
    for p in net.parameters():
        p.grad = None
    x.grad = None
    monkeypatch.setenv("NNDT_FUSED_MLP", "0")
    ref = net(x)                                   # nn.Sequential
    (ref * w).sum().backward()
    tol = dict(rtol=1e-9, atol=1e-10) if dtype == torch.float64 else dict(rtol=2e-3, atol=2e-4)
    torch.testing.assert_close(out, ref, **tol)
    torch.testing.assert_close(gx_fused, x.grad, **tol)
    for a, p in zip(g_fused, net.parameters()):
        scale = p.grad.abs().max().clamp_min(1e-6)
        assert ((a - p.grad).abs().max() / scale).item() < (1e-8 if dtype == torch.float64 else 2e-3)


def test_rl_problem_runs_fused_mlp_kernels_on_cuda():
    """The distributed-PPO trainers on CUDA: actor / critic forward + backward go through the fused MLP kernels
    (one DiNNO round of the RL problem, finite parameters afterwards)."""
    import networkx as nx
    from nn_distributed_training_b200.rl.consensus_ppo import DiNNOPPO
    from nn_distributed_training_b200.rl.dist_ppo import DistPPOProblem
    from nn_distributed_training_b200.rl.model import FFReLUNet
    from nn_distributed_training_b200.rl.simple_tag import SimpleTagEnv
    env = SimpleTagEnv(num_envs=8, num_good=1, num_adversaries=3, num_obstacles=8, max_cycles=40, device=DEV, seed=0)
    pr = DistPPOProblem(FFReLUNet([12, 64, 64, 64, 5]), FFReLUNet([12, 64, 64, 64, 1]), nx.wheel_graph(3), env,
                        timesteps_per_batch=400, max_timesteps_per_episode=40, gamma=0.99, n_updates_per_iteration=2, lr=3e-4,
                        clip=0.2, seed=0)
    conf = dict(max_rl_timesteps=800, ID=0, out_dir="/tmp/nndt_rl_test", writeout=False, rho_init=1.0, rho_scaling=1.0,
                primal_lr_start=3e-4, primal_lr_finish=1e-3, lr_decay_type="constant", persistant_primal_opt=False,
                primal_iterations=2, outer_iterations=10 ** 6)
    DiNNOPPO(pr, torch.device(DEV), conf).train()
    for m in pr.models.values():
        assert all(torch.isfinite(p).all() for p in m.parameters())


# ---- tensor-core density kernels against the bf16-faithful fp64 oracle ------------------------------------------------
LOSS_NAME = {"BCELoss": "BCE", "MSELoss": "MSE", "L1Loss": "L1"}


def _fused_density(L, B, M, h1=256, loss="BCE", net="fourier", seed=0):
    """A fused density problem of L nodes with M rows each and a different network per node."""
    from nn_distributed_training_b200.data.shards import Shard
    from nn_distributed_training_b200.models.relu_nn import FFReLUNet
    from nn_distributed_training_b200.problems import DistDensityProblem
    g = torch.Generator().manual_seed(seed)
    span = 1200.0 if net == "fourier" else 2.0          # the ReLU net takes normalised coordinates
    shards = [Shard((torch.rand(M, 2, generator=g) - 0.5) * span, (torch.rand(M, generator=g) < 0.3).float())
              for _ in range(L)]
    conf = {"problem_name": "d", "train_batch_size": B, "val_batch_size": 200,
            "metrics": ["forward_pass_count", "validation_loss", "consensus_error", "current_epoch"],
            "metrics_config": {"evaluate_frequency": 100}, "optimizer_config": {}}
    torch.manual_seed(seed)
    shape = [2, h1, 64, 64, 64, 1]
    base = FourierNet(shape, scale=0.05) if net == "fourier" else FFReLUNet(shape)
    lossf = {"BCE": torch.nn.BCELoss(), "MSE": torch.nn.MSELoss(), "L1": torch.nn.L1Loss()}[loss]
    pr = DistDensityProblem(nx.cycle_graph(L), base, lossf, shards, shards[0], DEV, conf, backend="fused", seed=3)
    assert pr.backend == "fused"
    for l in range(L):
        pr.arena.theta[l] *= 1.0 + 0.03 * l
    return pr


def _oracle(pr, l, call, rounding=True, cache=None):
    rows = ko.batch_rows(pr.shards.sizes, pr.train_batch_size, pr.seed, l, call, pr.placement.lo).to(DEV)
    return ko.mlp_bf16_faithful(pr.arena.theta[l], pr.base_model.spec, pr.shards.x[rows], pr.shards.y[rows],
                                LOSS_NAME[type(pr.base_loss).__name__], rounding=rounding, cache=cache)


def _assert_grad_row(got, gf, ge, spec):
    """Kernel gradient row against the faithful oracle ``gf`` with yardstick ``ge``.  The output-bias gradient
    mean(dL/dz) is a single number that the bf16 roundings barely touch (for L1 on the ReLU net, or on saturated BCE
    rows, it is the same number in both oracles), so it has no yardstick error to scale: it is held to fp32 accuracy
    on its own, every other tensor to the yardstick."""
    o9 = ko.slots(spec)[9][0]
    got = got.double().clone()
    torch.testing.assert_close(got[o9], gf[o9], rtol=1e-4, atol=1e-6)
    got[o9] = gf[o9]
    return ko.assert_close_to_oracle(got, gf, ge, ko.MLP_FRAC, spec=spec)


def _check_train_step(pr, tag):
    """One fused compute_grads() of every node against the faithful oracle on the rows it drew: gradient error at most
    MLP_FRAC x the faithful reference's own error against exact fp64, per tensor and per 16 x 8 block; same loss."""
    calls = pr.calls.copy()
    loss = pr.fused.compute_grads().clone()
    worst = 0.0
    for l in range(pr.placement.L):
        lf, gf, _ = _oracle(pr, l, int(calls[l]))
        ge = _oracle(pr, l, int(calls[l]), rounding=False)[1]
        rat = _assert_grad_row(pr.arena.grad[l], gf, ge, pr.base_model.spec)
        worst = max(worst, *(max(v) for v in rat.values()))
        torch.testing.assert_close(loss[l].double(), lf, rtol=1e-4, atol=1e-6)
    print(f"\nRATIO mlp_train {tag} call {int(calls[0])}: {worst:.2e}")


@pytest.mark.parametrize("h1", [64, 128, 256])
@pytest.mark.parametrize("L,B", [(4, 12500), (2, 20000)])
def test_train_kernel_production_partition_matches_oracle(L, B, h1):
    """dist_online_dense_PAPER's batch sizes: L x ceil(B / 128) tiles exceed the SMs, so a CTA accumulates several
    tiles (acc_store add), crosses node boundaries (flush + next slot), and in the partial second batch the CTAs whose
    tiles all lie past its end write zeros (!have_acc)."""
    pr = _fused_density(L, B, M=B + B // 2 + 1, h1=h1)
    assert pr.fused.G < L * -(-B // 128)
    for _ in range(2):
        _check_train_step(pr, f"L={L} B={B} h1={h1}")


@pytest.mark.parametrize("B", [1, 127, 128, 129, 1000])
def test_train_kernel_any_cta_count_matches_oracle(B):
    """The static (node, tile) partition over G CTAs, G from one CTA walking every tile of every node to more CTAs
    than tiles: the summed gradients agree across G up to fp32 reassociation and each matches the oracle.  CTAs never
    wait on each other, so every G is a valid launch."""
    L = 3
    pr = _fused_density(L, B, M=B + B // 2 + 1, h1=128)
    fz, spec = pr.fused, pr.base_model.spec
    I = L * -(-B // 128)
    Gs = sorted({1, 2, 7, I - 1, I, 132} - {0})
    for call in (0, 1):
        got = {}
        for G in Gs:
            S = -(-G // L) + 1
            gp = torch.zeros(L, S, fz.n_pad, device=DEV)
            lp = torch.zeros(L, S, device=DEV)
            fz.calls.fill_(call)
            fz.ext.MlpOp(dict(fz.base, train_ctas=G, S=S, grad_part=gp.data_ptr(), loss_part=lp.data_ptr())).train()
            got[G] = (gp.sum(1), lp.sum(1))
        for l in range(L):
            lf, gf, _ = _oracle(pr, l, call)
            ge = _oracle(pr, l, call, rounding=False)[1]
            g1 = got[Gs[0]][0][l]
            for G in Gs:
                g = got[G][0][l]
                for o, s in ko.slots(spec):
                    n = int(torch.tensor(s).prod())
                    torch.testing.assert_close(g[o: o + n], g1[o: o + n], rtol=1e-5,
                                               atol=1e-5 * g1[o: o + n].abs().max().item(), msg=f"G={G} slot {o}")
                _assert_grad_row(g, gf, ge, spec)
                torch.testing.assert_close(got[G][1][l].double(), lf, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("L", [1, 3, 8])
@pytest.mark.parametrize("M", [1, 127, 129, 10000, 50000])
def test_forward_kernel_matches_faithful_forward(M, L):
    """MlpForward over M rows: a partial last tile, one row, and more tiles than CTAs (the grid-stride loop).  The
    output's error against the faithful forward pass, as an RMS over all rows, is at most MLP_FRAC x the faithful
    pass's own error against exact fp64, and at most 0.5x in every 128-row tile (measured: 0.33 at worst, where one
    tile holds a few one-ulp bf16 rounding differences; a wrong tile is off by the size of the output).  The yardstick
    is measured on 8192 rows of the same input distribution, so it does not depend on M."""
    from nn_distributed_training_b200.ops.mlp_fused import MlpForward
    arena, _, spec = _arena([2, 256, 64, 64, 64, 1], 0.05, L)
    g = torch.Generator(device=DEV).manual_seed(M)
    x = (torch.rand(M, 2, device=DEV, generator=g) - 0.5) * 1500
    xc = (torch.rand(8192, 2, device=DEV, generator=g) - 0.5) * 1500
    fwd = MlpForward(arena, spec, L, torch.device(DEV))
    out = fwd(x).double()
    worst = 0.0
    for l in range(L):
        th = arena.theta[l]
        pf = ko.mlp_bf16_faithful(th, spec, x, torch.zeros(M, device=DEV), "MSE")[2]
        cal = (ko.mlp_bf16_faithful(th, spec, xc, xc[:, 0], "MSE", rounding=False)[2]
               - ko.mlp_bf16_faithful(th, spec, xc, xc[:, 0], "MSE")[2])
        yard = cal.pow(2).mean().sqrt()
        tiles = ko._block_errors(out[l] - pf, (128, 1)) / torch.tensor(
            [min(128, M - 128 * i) for i in range(-(-M // 128))], device=DEV).sqrt()
        worst = max(worst, (tiles.max() / yard).item())
        assert (out[l] - pf).pow(2).mean().sqrt() <= ko.MLP_FRAC * yard
        assert (tiles <= 0.5 * yard).all(), (l, (tiles.max() / yard).item())
    print(f"\nRATIO mlp_forward M={M} L={L}: {worst:.2e}")


@pytest.mark.parametrize("net,loss", [("fourier", "BCE"), ("fourier", "MSE"), ("fourier", "L1"),
                                      ("relu", "MSE"), ("relu", "L1")])
def test_train_kernel_specs_and_losses_match_oracle(net, loss):
    """Every network / loss pair the dispatcher accepts: FourierNet (sin_relu / sigmoid) and FFReLUNet([2, h, 64, 64,
    64, 1]) (relu / none), over an epoch end with a partial batch."""
    pr = _fused_density(3, 300, M=451, h1=128, loss=loss, net=net)
    for _ in range(3):
        _check_train_step(pr, f"{net}/{loss}")


def test_train_kernel_saturated_bce_rows():
    """Rows whose output pre-activation z lies in [20, 40], where fp32 rounds the sigmoid to 1.  Intended behaviour of
    the fused kernel: the gradient is that of the exact loss, dL/dz = p - y (so a y = 0 row still pulls z down), and the
    reported loss is torch's fp32 definition, log clamped at -100.  The torch backend differs on these rows: its fp32
    autograd returns a zero gradient there (tests/test_kernel_oracles.py::test_saturated_bce_rows_in_fp32_autograd)."""
    pr = _fused_density(3, 300, M=451, h1=128)
    o_b4 = ko.slots(pr.base_model.spec)[9][0]
    pr.arena.theta[:, o_b4] = 30.0
    for _ in range(2):
        calls = pr.calls.copy()
        loss = pr.fused.compute_grads().clone()
        for l in range(3):
            cache = {}
            lf, gf, p = _oracle(pr, l, int(calls[l]), cache=cache)
            ge = _oracle(pr, l, int(calls[l]), rounding=False)[1]
            z = torch.logit(p)
            assert ((z > 20) & (z < 40)).all()
            _assert_grad_row(pr.arena.grad[l], gf, ge, pr.base_model.spec)
            rows = ko.batch_rows(pr.shards.sizes, 300, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            y = pr.shards.y[rows]
            p32 = torch.sigmoid(z.float())
            assert (p32 == 1.0).all()
            l32 = -(y * torch.log(p32).clamp_min(-100) + (1 - y) * torch.log(1 - p32).clamp_min(-100)).mean()
            torch.testing.assert_close(loss[l], l32, rtol=1e-5, atol=0)
            assert lf.item() < 0.5 * l32.item()          # the exact loss is far below the clamped one
