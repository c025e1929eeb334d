"""GPU tests of the float64 density MLP kernels (csrc/mlp_f64.cu): against the exact fp64 oracle, across launch widths,
bitwise determinism, and whole fp64 training runs against autograd + the PyTorch consensus ops."""
import copy

import networkx as nx
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.models import FourierNet
from nn_distributed_training_b200.optimizers import DiNNO, DSGD, DSGT

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOSS_NAME = {"BCELoss": "BCE", "MSELoss": "MSE", "L1Loss": "L1"}
# The kernel's error may be at most this fraction of the error of the same math accumulated in fp32, per tensor and
# per 16 x 8 block.  fp64 accumulation in a different order should measure about 1e-8; a zeroed or doubled tile
# measures far above 1.
F64_FRAC = 1e-4
CONF = {"problem_name": "d", "val_batch_size": 200,
        "metrics": ["forward_pass_count", "validation_loss", "consensus_error", "current_epoch"],
        "metrics_config": {"evaluate_frequency": 3}}


def _density(L, B, M, h1=256, loss="BCE", net="fourier", backend="fused", seed=0, opt_conf=None, perturb=True):
    """A float64 density problem of L nodes with M rows each and a different network per node."""
    from nn_distributed_training_b200.data.shards import Shard
    from nn_distributed_training_b200.models.relu_nn import FFReLUNet
    from nn_distributed_training_b200.problems import DistDensityProblem
    g = torch.Generator().manual_seed(seed)
    span = 1200.0 if net == "fourier" else 2.0          # the ReLU net takes normalised coordinates
    shards = [Shard(((torch.rand(M, 2, generator=g, dtype=torch.float64) - 0.5) * span),
                    (torch.rand(M, generator=g) < 0.3).double()) for _ in range(L)]
    val = Shard(((torch.rand(300, 2, generator=g, dtype=torch.float64) - 0.5) * span),
                (torch.rand(300, generator=g) < 0.3).double())
    conf = dict(CONF, train_batch_size=B, optimizer_config=opt_conf or {})
    torch.manual_seed(seed)
    shape = [2, h1, 64, 64, 64, 1]
    base = (FourierNet(shape, scale=0.05, dtype=torch.float64) if net == "fourier"
            else FFReLUNet(shape, dtype=torch.float64))
    lossf = {"BCE": torch.nn.BCELoss(), "MSE": torch.nn.MSELoss(), "L1": torch.nn.L1Loss()}[loss]
    pr = DistDensityProblem(nx.cycle_graph(L), base, lossf, shards, val, DEV, conf, backend=backend, seed=3)
    assert pr.dtype == torch.float64
    if perturb:
        # not affine in l: on a cycle an affine perturbation makes delta of the interior nodes exactly 0, and a result
        # that then hangs on the sign of a round-off residue (tests/test_consensus_oracle.py)
        for l in range(L):
            pr.arena.theta[l] *= 1.0 + 0.03 * l * l
    return pr


def _oracle(pr, l, call, accum=torch.float64):
    rows = ko.batch_rows(pr.shards.sizes, pr.train_batch_size, pr.seed, l, call, pr.placement.lo).to(DEV)
    return ko.mlp_bf16_faithful(pr.arena.theta[l], pr.base_model.spec, pr.shards.x[rows], pr.shards.y[rows],
                                LOSS_NAME[type(pr.base_loss).__name__], rounding=False, accum=accum)


def _assert_grad_row(got, pr, l, call):
    """Gradient row against the exact oracle, yardstick: the same math accumulated in fp32.  The output-bias gradient
    mean(dL/dz) is one sum the yardstick can get exactly right, so it is held to 1e-12 on its own."""
    spec = pr.base_model.spec
    lf, ge, _ = _oracle(pr, l, call)
    gy = _oracle(pr, l, call, accum=torch.float32)[1].double()
    o9 = ko.slots(spec)[9][0]
    got = got.clone()
    torch.testing.assert_close(got[o9], ge[o9], rtol=1e-12, atol=1e-15)
    got[o9] = ge[o9]
    return lf, ko.assert_close_to_oracle(got, ge, gy, F64_FRAC, spec=spec)


def _check_train_step(pr, tag):
    calls = pr.calls.copy()
    loss = pr.fused.compute_grads().clone()
    worst = 0.0
    for l in range(pr.placement.L):
        lf, rat = _assert_grad_row(pr.arena.grad[l], pr, l, int(calls[l]))
        worst = max(worst, *(max(v) for v in rat.values()))
        torch.testing.assert_close(loss[l], lf, rtol=1e-12, atol=0)
    print(f"\nRATIO mlp_f64 {tag} call {int(calls[0])}: {worst:.2e}")


@pytest.mark.parametrize("h1", [64, 128, 256])
@pytest.mark.parametrize("L,B", [(4, 12500), (2, 20000)])
def test_f64_train_kernel_production_partition_matches_oracle(L, B, h1):
    """dist_online_dense_PAPER's batch sizes: a cluster walks many tiles and crosses node boundaries, and in the
    partial second batch some clusters own only tiles past its end."""
    pr = _density(L, B, M=B + B // 2 + 1, h1=h1)
    assert pr.backend == "fused" and pr.fused.G < L * -(-B // 32)
    for _ in range(2):
        _check_train_step(pr, f"L={L} B={B} h1={h1}")


@pytest.mark.parametrize("B", [1, 31, 32, 33, 1000])
def test_f64_train_kernel_partial_batches_match_oracle(B):
    pr = _density(3, B, M=B + B // 2 + 1, h1=128)
    for _ in range(3):
        _check_train_step(pr, f"B={B}")


@pytest.mark.parametrize("net,loss", [("fourier", "BCE"), ("fourier", "MSE"), ("fourier", "L1"),
                                      ("relu", "MSE"), ("relu", "L1")])
def test_f64_train_kernel_specs_and_losses_match_oracle(net, loss):
    pr = _density(3, 300, M=451, h1=128, loss=loss, net=net)
    for _ in range(3):
        _check_train_step(pr, f"{net}/{loss}")


def _launch(fz, G, call):
    L = fz.L
    S = 2 * (-(-G // L) + 1)
    gp = torch.zeros(L, S, fz.n_pad, dtype=torch.float64, device=DEV)
    lp = torch.zeros(L, S, dtype=torch.float64, device=DEV)
    fz.calls.fill_(call)
    fz.ext.MlpOp(dict(fz.base, train_ctas=G, S=S, grad_part=gp.data_ptr(), loss_part=lp.data_ptr())).train()
    return gp, lp


@pytest.mark.parametrize("B", [1, 33, 1000])
def test_f64_train_kernel_any_cluster_count_matches_oracle(B):
    """The static (node, tile) partition over G clusters, from one cluster walking every tile of every node to more
    clusters than tiles (and than fit on the GPU at once): each width matches the oracle, and the summed gradients of
    all widths agree to fp64 reassociation."""
    L = 3
    pr = _density(L, B, M=B + B // 2 + 1, h1=128)
    fz = pr.fused
    I = L * -(-B // 32)
    Gs = sorted({1, 2, 7, I - 1, I, 66, 132} - {0})
    for call in (0, 1):
        got = {G: [t.sum(1) for t in _launch(fz, G, call)] for G in Gs}
        for l in range(L):
            g1 = got[Gs[0]][0][l]
            for G in Gs:
                g = got[G][0][l]
                torch.testing.assert_close(g, g1, rtol=1e-12, atol=1e-14 * g1.abs().max().item(), msg=f"G={G}")
                lf, _ = _assert_grad_row(g, pr, l, call)
                torch.testing.assert_close(got[G][1][l], lf, rtol=1e-12, atol=0)


def test_f64_train_kernel_is_deterministic():
    """No atomics: two launches on the same inputs give bitwise-equal partial rows and losses."""
    pr = _density(4, 12500, M=15000, h1=256)
    fz = pr.fused
    for call in (0, 1):
        a = _launch(fz, fz.G, call)
        b = _launch(fz, fz.G, call)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("L", [1, 3, 8])
@pytest.mark.parametrize("M", [1, 127, 129, 10000, 50000])
def test_f64_forward_kernel_matches_exact_oracle(M, L):
    """MlpForward in float64 over M rows (partial last tile, one row, more tiles than clusters): every output within
    1e-12 of the exact oracle."""
    from nn_distributed_training_b200.ops.mlp_fused import MlpForward
    from nn_distributed_training_b200.parallel.arena import FlatLayout, NodeArena
    torch.manual_seed(M + L)
    shape = [2, 256, 64, 64, 64, 1]
    base = FourierNet(shape, scale=0.05, dtype=torch.float64)
    arena = NodeArena(FlatLayout.from_module(base), L, DEV, torch.float64)
    for l in range(L):
        arena.attach(l, FourierNet(shape, scale=0.05, dtype=torch.float64).to(DEV))
    g = torch.Generator(device=DEV).manual_seed(M)
    x = (torch.rand(M, 2, device=DEV, generator=g, dtype=torch.float64) - 0.5) * 1500
    out = MlpForward(arena, base.spec, L, torch.device(DEV))(x)
    assert out.dtype == torch.float64
    for l in range(L):
        p = ko.mlp_bf16_faithful(arena.theta[l], base.spec, x, torch.zeros(M, device=DEV), "MSE", rounding=False)[2]
        assert (out[l] - p).abs().max().item() <= 1e-12


def test_f64_fused_grads_match_autograd_per_step():
    """compute_grads() of the fused and the autograd path on the same parameters: fp64 round-off per step."""
    fused = _density(3, 1000, M=1500)
    ref = _density(3, 1000, M=1500, backend="torch")
    assert fused.backend == "fused" and ref.backend == "torch"
    ref.arena.theta.copy_(fused.arena.theta)
    for _ in range(4):
        lf, lr = fused.compute_grads().clone(), ref.compute_grads().clone()
        torch.testing.assert_close(lf, lr, rtol=1e-9, atol=1e-12)
        torch.testing.assert_close(fused.arena.grad, ref.arena.grad, rtol=1e-9, atol=1e-11)
    assert (fused.calls == ref.calls).all()


DINNO = {"alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.01, "outer_iterations": 7,
         "primal_iterations": 2, "primal_optimizer": "adam", "persistant_primal_opt": False,
         "primal_lr_start": 0.005, "primal_lr_finish": 0.0005, "lr_decay_type": "log", "profile": False}
DSGD_C = {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.01, "outer_iterations": 7, "profile": False}
DSGT_C = {"alg_name": "dsgt", "alpha": 0.02, "init_grads": True, "outer_iterations": 7, "profile": False}


@pytest.mark.parametrize("cls,conf", [(DiNNO, DINNO), (DSGD, DSGD_C), (DSGT, DSGT_C)])
def test_f64_fused_density_training_matches_torch_fp64(cls, conf):
    """Fused fp64 forward/backward and fp64 consensus kernels under CUDA graphs against autograd and the PyTorch
    consensus ops in float64: agreement to fp64 round-off over the whole run.  The nodes start from a perturbation that
    is not affine in l; an affine one makes delta of the interior nodes of the cycle exactly 0 in exact arithmetic,
    so on coordinates without a loss gradient Adam steps by +-lr on the sign of a round-off residue, and the run
    depended on how delta was rounded rather than on the kernels (it ended 8.5e-5 apart while the exchange of the
    PyTorch ops took sums instead of per-neighbor differences)."""
    a = _density(4, 500, M=700, opt_conf=copy.deepcopy(conf))
    b = _density(4, 500, M=700, backend="torch", opt_conf=copy.deepcopy(conf))
    b.arena.theta.copy_(a.arena.theta)
    opt = cls(a, DEV, dict(copy.deepcopy(conf), consensus_backend="auto"))
    assert opt._use_engine()
    opt.train()
    cls(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch")).train()
    rel = ((a.arena.theta - b.arena.theta).norm() / b.arena.theta.norm()).item()
    assert rel < 1e-8, rel
    assert a.forward_cnt == b.forward_cnt
    torch.testing.assert_close(a.metrics["validation_loss"][-1], b.metrics["validation_loss"][-1], rtol=1e-9, atol=0)


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
            "metrics": ["forward_pass_count", "train_loss_moving_average", "validation_loss", "consensus_error",
                        "current_epoch"],
            "metrics_config": {"evaluate_frequency": 4, "tloss_decay": 0.2, "mesh_only_at_end": True},
            "optimizer_config": opt_conf}
    torch.manual_seed(0)
    base = FourierNet([2, 256, 64, 64, 64, 1], scale=0.05, dtype=torch.float64)
    return DistOnlineDensityProblem(base, torch.nn.BCELoss(), train, val, DEV, conf, backend=backend, seed=5)


def test_f64_online_density_training_matches_torch_fp64(tmp_path):
    """The online problem (dynamic graph, sliding-window stream with several window switches) in float64: the in-kernel
    sampler draws the rows the Python schedule draws, and the losses agree to fp64 round-off."""
    oc = {"alg_name": "dinno", "rho_init": 0.3, "rho_scaling": 1.0004, "outer_iterations": 9, "primal_iterations": 3,
          "primal_optimizer": "adam", "persistant_primal_opt": False, "primal_lr_start": 0.001,
          "primal_lr_finish": 0.0001, "lr_decay_type": "log", "profile": False}
    fused = _online_problem("fused", str(tmp_path), oc)
    ref = _online_problem("torch", str(tmp_path), oc)
    assert fused.backend == "fused" and fused.dtype == torch.float64
    ref.arena.theta.copy_(fused.arena.theta)
    DiNNO(fused, DEV, oc).train()
    DiNNO(ref, DEV, dict(oc, consensus_backend="torch")).train()
    assert (fused.positions() == ref.positions()).all()
    assert fused.forward_cnt == ref.forward_cnt
    assert len(fused.metrics["validation_loss"]) == len(ref.metrics["validation_loss"]) == 3
    for key in ("validation_loss", "train_loss_moving_average"):
        torch.testing.assert_close(fused.metrics[key][-1], ref.metrics[key][-1], rtol=1e-9, atol=1e-12)
    rel = ((fused.arena.theta - ref.arena.theta).norm() / ref.arena.theta.norm()).item()
    assert rel < 1e-8, rel


@pytest.mark.parametrize("cls,conf", [(DiNNO, dict(DINNO, persistant_primal_opt=True, outer_iterations=6)),
                                      (DSGT, dict(DSGT_C, outer_iterations=6))])
def test_f64_density_checkpoint_resume_is_bit_exact(tmp_path, cls, conf):
    """Crash after an odd round, resume in a fresh problem and optimizer on the fused fp64 path: parameters equal the
    uninterrupted run bit for bit."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    full = _density(4, 300, M=500, opt_conf=conf)
    cls(full, DEV, copy.deepcopy(conf)).train()
    first = _density(4, 300, M=500, opt_conf=conf)
    o1 = cls(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3
    o1.train()
    assert o1.k == 3
    second = _density(4, 300, M=500, opt_conf=conf)
    o2 = cls(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert second.forward_cnt == full.forward_cnt


def test_f64_density_auto_backend_selects_fused(capsys):
    pr = _density(3, 100, M=200, backend="auto")
    assert pr.backend == "fused"
    assert "WARNING" not in capsys.readouterr().out


def test_f64_fused_backend_rejects_unsupported_shape():
    from nn_distributed_training_b200.data.shards import Shard
    from nn_distributed_training_b200.problems import DistDensityProblem
    x = torch.rand(100, 2, dtype=torch.float64)
    shards = [Shard(x, (x[:, 0] > 0.5).double()) for _ in range(3)]
    conf = dict(CONF, train_batch_size=50, optimizer_config={})
    base = FourierNet([2, 96, 64, 64, 64, 1], scale=0.05, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="fused"):
        DistDensityProblem(nx.cycle_graph(3), base, torch.nn.BCELoss(), shards, shards[0], DEV, conf, backend="fused")
