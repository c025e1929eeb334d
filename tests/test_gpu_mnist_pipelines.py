"""The staged and host-fed input pipelines for every MNIST training kernel and both row types.

``input_pipeline: auto`` resolves to ``staged`` whenever the round is captured, so production training reads its
batches through ``gather_rows_kernel`` and the kernels' direct path (``direct = 1``: row ``l * batch + t`` of the
staging set, the drawn batch size from ``direct_bs``), not through the in-kernel sampler.  Both pipelines draw the same
rows from the same stateless sampler, so a run must train exactly like the resident one, bit for bit."""
import networkx as nx
import pytest
import torch

from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.optimizers import DiNNO
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DINNO = {"alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.01, "outer_iterations": 12,
         "primal_iterations": 2, "primal_optimizer": "adam", "persistant_primal_opt": False,
         "primal_lr_start": 0.005, "primal_lr_finish": 0.0005, "lr_decay_type": "log", "profile": False}
# kernel -> (MNISTConvNet shape, dtype, batch, extra problem conf); every shard holds 2.5 batches, so the rounds draw
# partial batches and wrap epochs
KERNELS = {"batch_split_f32": ((3, 5, 64), torch.float32, 100, {"samples_per_cta": 7}),
           "generic_f64": ((3, 5, 64), torch.float64, 100, {}),
           "generic_f32_2x5x32": ((2, 5, 32), torch.float32, 32, {}),
           "cl64_f64": ((3, 5, 64), torch.float64, 64, {}),
           "tc_f32": ((3, 5, 64), torch.float32, 64, {})}


def _problem(kernel, float_rows, pipeline, N=4):
    shape, dtype, B, extra = KERNELS[kernel]
    M = B * 5 // 2
    data = synthetic_mnist(M * N, seed=3)
    shards = [data.select(torch.arange(i * M, (i + 1) * M)) for i in range(N)]
    if float_rows:
        shards = [Shard(s.inputs(torch.arange(len(s)), torch.float32), s.y) for s in shards]
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": ["forward_pass_count"],
            "metrics_config": {"evaluate_frequency": 1000}, "optimizer_config": dict(DINNO),
            "input_pipeline": pipeline, **extra}
    torch.manual_seed(0)
    pr = DistMNISTProblem(nx.cycle_graph(N), MNISTConvNet(*shape, dtype=dtype), torch.nn.NLLLoss(), shards,
                          synthetic_mnist(16, seed=4), DEV, conf, backend="fused", seed=7)
    fz = pr.fused
    which = {"batch_split_f32": not fz.generic and not fz.tc and fz.spb == 7,
             "generic_f64": fz.generic and not fz.cl64, "generic_f32_2x5x32": fz.generic,
             "cl64_f64": fz.cl64, "tc_f32": fz.tc}
    assert which[kernel], fz.kernel_name
    assert fz.x_is_u8 != float_rows
    return pr


@pytest.mark.parametrize("pipeline", ["staged", "host"])
@pytest.mark.parametrize("float_rows", [False, True], ids=["u8", "f32"])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_pipeline_trains_like_resident(kernel, float_rows, pipeline):
    """DiNNO for 5 + 4 rounds of 2 primal steps: ``theta``, ``forward_cnt`` and the draw counters equal the resident
    run's bit for bit.  f32 rows are 3136 bytes, the only row size that takes the gather's tail loop."""
    outs = []
    for pl in ("resident", pipeline):
        pr = _problem(kernel, float_rows, pl)
        opt = DiNNO(pr, DEV, dict(DINNO))
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), pr.forward_cnt, pr.calls.copy()))
        if pl == "host":
            assert torch.isfinite(pr.fused.loss_host).all() and pr.fused.loss_host.abs().sum() > 0
    assert torch.equal(outs[0][0], outs[1][0])
    assert outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()
