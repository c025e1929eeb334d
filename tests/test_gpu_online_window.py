"""The rows the density training kernels draw from the online sliding-window stream (ops/csrc/sampler.cuh,
``stream_row`` over ``data.sampler.window_table``), in float32 (csrc/mlp_tc.cu) and float64 (csrc/mlp_f64.cu).

Each node's draw counter is set directly, so one launch reaches any point of the stream: a batch inside one window,
across a boundary, over several windows, across the period wrap, an epoch's partial last batch, positions past 2^32.
The oracle is the node's shard offset plus ``OnlineWindowSchedule.indices`` at the batch's stream position, keyed by
the global node id (what ``DistOnlineDensityProblem._draw_indices`` draws); the gradient row and loss of the launch
are compared with ``kernel_oracles.mlp_bf16_faithful`` on those rows.  The shard rows are random, so a batch off by
one row changes the gradient by O(1) of the yardsticks."""
import numpy as np
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.data.sampler import OnlineWindowSchedule
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.models import FourierNet

from window_oracle import CASES, schedule_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 5
F64_FRAC = 1e-4          # as tests/test_gpu_mlp_f64.py
TILE = {torch.float32: 128, torch.float64: 32}


@pytest.fixture(scope="module", autouse=True)
def _fp32_references():
    with ko.fp32_references():
        yield


class _Stream:
    """Stand-in for ``OnlineTrajectoryLidarDataset``: T scans of S random rows, streamed through windows of Wn scans."""

    def __init__(self, T, S, Wn, dtype, seed):
        g = torch.Generator().manual_seed(seed)
        self.shard = Shard(((torch.rand(T * S, 2, generator=g, dtype=torch.float64) - 0.5) * 1200).to(dtype),
                           (torch.rand(T * S, generator=g) < 0.3).to(dtype))
        self.schedule = OnlineWindowSchedule(T, S, Wn)
        self.scan_locs = np.random.default_rng(seed).uniform(-10, 10, size=(T, 2))

    def pos_after(self, draws):
        return self.scan_locs[self.schedule.scan_cursor_at(draws), :]

    def __len__(self):
        return len(self.shard.y)


def _problem(geoms, B, dtype):
    from nn_distributed_training_b200.problems import DistOnlineDensityProblem
    train = [_Stream(T, S, Wn, dtype, seed=i) for i, (T, S, Wn) in enumerate(geoms)]
    val = _Stream(4, 25, 2, dtype, seed=99).shard
    conf = {"problem_name": "w", "train_batch_size": B, "val_batch_size": 100, "comm_radius": 1e6,
            "dynamic_graph": True, "save_models": False,
            "metrics": ["forward_pass_count", "validation_loss", "consensus_error", "current_epoch"],
            "metrics_config": {"evaluate_frequency": 100}, "optimizer_config": {}}
    torch.manual_seed(0)
    base = FourierNet([2, 128, 64, 64, 64, 1], scale=0.05, dtype=dtype)
    pr = DistOnlineDensityProblem(base, torch.nn.BCELoss(), train, val, DEV, conf, backend="fused", seed=SEED)
    assert pr.backend == "fused" and pr.fused.win_table is not None and pr.dtype == dtype
    for l in range(pr.placement.L):
        pr.arena.theta[l] *= 1.0 + 0.03 * l * l
    return pr


def _launch(fz, calls, G, node0=0):
    """One training launch over G CTAs (float32) or G 2-CTA clusters (float64) at the given draw counters."""
    L = fz.L
    S = -(-G // L) + 1
    if fz.dtype == torch.float64:
        S *= 2
    gp = torch.zeros(L, S, fz.n_pad, dtype=fz.dtype, device=DEV)
    lp = torch.zeros(L, S, dtype=fz.dtype, device=DEV)
    fz.calls.copy_(torch.tensor(calls, dtype=torch.int32))
    fz.ext.MlpOp(dict(fz.base, train_ctas=G, S=S, grad_part=gp.data_ptr(), loss_part=lp.data_ptr(), node0=node0)).train()
    return gp.sum(1), lp.sum(1)


def _rows(pr, l, call, node0):
    sizes = pr.shards.sizes
    off = sum(int(m) for m in sizes[:l])
    m = int(sizes[l])
    return off + torch.as_tensor(schedule_rows(pr._datasets[l].schedule, m, pr.train_batch_size, call, SEED, node0 + l))


def _check(pr, l, rows, grad, loss):
    """Gradient row and loss of node l against the faithful oracle on ``rows``, with each dtype's yardstick."""
    spec = pr.base_model.spec
    rows = rows.to(DEV)
    x, y = pr.fused.x[rows], pr.fused.y[rows]
    th = pr.arena.theta[l]
    o9 = ko.slots(spec)[9][0]
    got = grad.double().clone()
    if pr.dtype == torch.float32:
        lf, gf, _ = ko.mlp_bf16_faithful(th, spec, x, y, "BCE")
        ge = ko.mlp_bf16_faithful(th, spec, x, y, "BCE", rounding=False)[1]
        torch.testing.assert_close(got[o9], gf[o9], rtol=1e-4, atol=1e-6)
        got[o9] = gf[o9]
        ko.assert_close_to_oracle(got, gf, ge, ko.MLP_FRAC, spec=spec)
        torch.testing.assert_close(loss.double(), lf, rtol=1e-4, atol=1e-6)
    else:
        lf, ge, _ = ko.mlp_bf16_faithful(th, spec, x, y, "BCE", rounding=False)
        gy = ko.mlp_bf16_faithful(th, spec, x, y, "BCE", rounding=False, accum=torch.float32)[1].double()
        torch.testing.assert_close(got[o9], ge[o9], rtol=1e-12, atol=1e-15)
        got[o9] = ge[o9]
        ko.assert_close_to_oracle(got, ge, gy, F64_FRAC, spec=spec)
        torch.testing.assert_close(loss, lf, rtol=1e-12, atol=0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_window_draws_match_schedule(case, dtype):
    """Every launch of the case at G = 1, 2, the problem's own width and more CTAs than tiles (so one batch's window
    boundaries fall in different CTAs), with the global ids starting at node0 = 0 and at node0 = 7."""
    geoms, B, launches = CASES[case]
    pr = _problem(geoms, B, dtype)
    fz = pr.fused
    tiles = fz.L * -(-B // TILE[dtype])
    paper = B >= 10000
    Gs = sorted({1, fz.G} if paper else {1, 2, fz.G, tiles + 5})
    for i, calls in enumerate(launches):
        for node0 in ((0, 7) if i == 1 else (0,)):
            rows = [_rows(pr, l, calls[l], node0) for l in range(fz.L)]
            for G in Gs:
                grad, loss = _launch(fz, calls, G, node0)
                for l in range(fz.L):
                    try:
                        _check(pr, l, rows[l], grad[l], loss[l])
                    except AssertionError as e:
                        raise AssertionError(f"{case} launch {calls} node {l} G={G} node0={node0}: {e}") from None


def test_window_stream_of_more_than_64_windows_is_refused():
    """K = 64 windows per period is the table's capacity (drawn correctly in the case "k64"); K = 65 is refused when
    the fused engine is built."""
    with pytest.raises(RuntimeError, match="more than 64 windows"):
        _problem([(20, 50, 3), (130, 3, 2)], 50, torch.float32)
