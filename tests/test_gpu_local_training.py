"""The fused solo / centralized baselines (``ops/local_train.py``) on the GPU.

* ``local_step_kernel`` one launch at a time against the float64 oracle of ``tests/local_train_oracle.py``, to the
  per-coordinate bound ``16 u x err`` of ``tests/test_gpu_consensus_kernels.py``; nodes at their budget bitwise
  untouched, padding left at 0.
* Whole runs against torch.optim fed the same batches (``HostTwinTrainer``): float64 to 1e-9 relative after one step
  and 1e-8 over the run; float32 MNIST within 4x the error of the torch float32 path against the float64 oracle;
  float32 density within the bf16 tolerance of ``tests/test_gpu_mlp.py``.
* Determinism, graph replay against eager launches, and the ``solo_results.pt`` of the online-density runner."""
import copy
import os

import numpy as np
import pytest
import torch
import yaml

import consensus_oracle as co
import local_train_oracle as lto
from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.sampler import BatchSchedule
from nn_distributed_training_b200.data.shards import Shard
from nn_distributed_training_b200.models import FourierNet, MNISTConvNet
from nn_distributed_training_b200.ops import load_ext, local_train
from nn_distributed_training_b200.problems.base import sum_of_batch_means

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
C = 16
SEED = 11
NPDT = {torch.float32: np.float32, torch.float64: np.float64}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


# ------------------------------------------------------------------------------------ one launch ----
def _launch_state(L, S, n, n_pad, dtype, seed, calls, budget):
    g = torch.Generator().manual_seed(seed)
    def rows(*shape, scale=1.0):
        t = torch.zeros(*shape, n_pad, dtype=torch.float64)
        t[..., :n] = torch.randn(*shape, n, generator=g, dtype=torch.float64) * scale
        return t.to(dtype).to(DEV)
    return dict(theta=rows(L), grad_part=rows(L, S, scale=0.3), m=rows(L, scale=0.01),
                v=rows(L, scale=1e-3).abs(), calls=torch.tensor(calls, dtype=torch.int32, device=DEV),
                budget=torch.tensor(budget, dtype=torch.int32, device=DEV),
                arrive=torch.zeros(L, dtype=torch.int32, device=DEV))


def _op(st, opt, lr, S, n_pad):
    ext = load_ext(required=True)
    d = dict(L=st["theta"].shape[0], n_pad=n_pad, S=S, theta=st["theta"].data_ptr(),
             grad_part=st["grad_part"].data_ptr(), calls=st["calls"].data_ptr(), budget=st["budget"].data_ptr(),
             arrive=st["arrive"].data_ptr(), m=st["m"].data_ptr(), v=st["v"].data_ptr(), local_lr=lr,
             opt={"sgd": 0, "adam": 1, "adamw": 2}[opt])
    return (ext.LocalStepOpF32 if st["theta"].dtype == torch.float32 else ext.LocalStepOpF64)(d)


def _np(st):
    return {k: v.double().cpu().numpy() if v.is_floating_point() else v.cpu().numpy() for k, v in st.items()}


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("opt", ["sgd", "adam", "adamw"])
@pytest.mark.parametrize("S", [1, 2, 4, 13])
@pytest.mark.parametrize("n,n_pad", [(1001, 1024), (150_000, 150_016)], ids=["padded", "grid_stride"])
def test_local_step_matches_oracle(dtype, opt, S, n, n_pad):
    """Four nodes: two below budget (one at its first step), one at its budget, one with a budget of 0.  Three launches:
    the second and third also reach the budgets on the device."""
    L, lr = 4, 3e-3
    st = _launch_state(L, S, n, n_pad, dtype, seed=S + 7 * n, calls=[0, 5, 2, 0], budget=[3, 7, 2, 0])
    op = _op(st, opt, lr, S, n_pad)
    u = co.unit_roundoff(NPDT[dtype])
    for launch in range(3):
        before = _np(st)
        op.step()
        torch.cuda.synchronize()
        after = _np(st)
        want, err = lto.local_step(before, opt=opt, lr=lr, u=u, dtype=NPDT[dtype])
        for key in ("theta", "m", "v") if opt != "sgd" else ("theta",):
            co.check(f"launch {launch} {key}", after[key], want[key], err[key], C)
            assert (after[key][:, n:] == 0).all(), f"padding of {key} written"
        for i in range(L):
            if before["calls"][i] >= before["budget"][i]:
                for key in ("theta", "m", "v"):
                    assert np.array_equal(after[key][i], before[key][i]), (launch, i, key)
        assert np.array_equal(after["calls"], want["calls"]), (launch, after["calls"], want["calls"])
        assert (after["arrive"] == 0).all()
        if opt == "sgd":
            assert np.array_equal(after["m"], before["m"]) and np.array_equal(after["v"], before["v"])
    assert st["calls"].tolist() == [3, 7, 2, 0]


# ----------------------------------------------------------------------------------- MNIST solo ----
def _mnist(sizes, dtype, seed=0):
    shards = [synthetic_mnist(m, seed=100 + g) for g, m in enumerate(sizes)]
    val = synthetic_mnist(150, seed=1)
    torch.manual_seed(seed)
    return MNISTConvNet(3, 5, 64, dtype=dtype), torch.nn.NLLLoss(), shards, val


def _mnist_trainer(base, loss, shards, val, B, epochs, opt="adam", lr=2e-3):
    pr = local_train.build_problem("mnist", base, loss, shards, val, DEV, B, 50, SEED)
    tr = local_train.LocalTrainer(pr, opt, lr, local_train.epoch_budgets(pr.node_sizes, B, epochs))
    return pr, tr


def _oracles(base, loss, shards, B, opt="adam", lr=2e-3, dtype=None, squeeze=False):
    out = []
    for g, s in enumerate(shards):
        m = copy.deepcopy(base).to(DEV)
        if dtype is not None:
            m = m.to(dtype)
        sh = Shard(s.x.to(DEV), s.y.to(DEV), s.norm)
        out.append(lto.HostTwinTrainer(m, loss, sh, B, opt, lr, SEED, g, squeeze=squeeze))
    return out


def _torch_mnist_eval(model, val, vb):
    """What ``dist_mnist_ex.train_solo`` reports for ``model``."""
    dtype = next(model.parameters()).dtype
    v = Shard(val.x.to(DEV), val.y.to(DEV), val.norm)
    loss, correct = 0.0, 0
    with torch.no_grad():
        for a in range(0, len(v), vb):
            idx = torch.arange(a, min(len(v), a + vb), device=DEV)
            out = model(v.inputs(idx, dtype))
            loss += torch.nn.functional.nll_loss(out, v.targets(idx)).item()
            correct += out.argmax(1).eq(v.targets(idx)).sum().item()
    return loss / len(v), correct / len(v)


@pytest.mark.parametrize("B,sizes,kernel", [(64, [150, 97, 77], "cl64"), (100, [230, 150, 61], "generic")])
def test_fp64_solo_mnist_matches_autograd(B, sizes, kernel):
    """The paper net in float64 at batch 64 (cluster kernel) and 100 (generic kernel), unequal shards with a partial
    last batch (the third node's shard at batch 100 is smaller than one batch)."""
    base, loss, shards, val = _mnist(sizes, torch.float64)
    pr, tr = _mnist_trainer(base, loss, shards, val, B, epochs=2)
    assert bool(pr.fused.cl64) == (kernel == "cl64") and pr.fused.generic
    refs = _oracles(base, loss, shards, B)
    tr.run(1)
    for g, r in enumerate(refs):
        r.run(1)
        assert _rel(lto.flat(pr.models[g]), lto.flat(r.model)) < 1e-9, g
    tr.run(tr.total - 1)
    budgets = local_train.epoch_budgets(sizes, B, 2)
    assert tr.steps_taken() == budgets
    for g, r in enumerate(refs):
        r.run(budgets[g] - 1)
        assert _rel(lto.flat(pr.models[g]), lto.flat(r.model)) < 1e-8, g

    conf = dict(optimizer="adam", lr=2e-3, epochs=2, train_batch_size=B, val_batch_size=50)
    res = local_train.solo_mnist(base, loss, shards, val, DEV, conf, seed=SEED)
    assert sorted(res) == list(range(len(sizes)))
    for g, r in enumerate(refs):
        vl, acc = _torch_mnist_eval(r.model, val, 50)
        assert isinstance(res[g]["validation_loss"], float) and isinstance(res[g]["validation_accuracy"], float)
        assert res[g]["validation_loss"] == pytest.approx(vl, rel=1e-8)
        assert res[g]["validation_accuracy"] == acc


def test_fp32_solo_mnist_within_4x_of_torch_fp32():
    """Float32 fused (the paper net at batch 64: the tensor-core cluster kernel) against the float64 oracle: no further
    off than torch.optim in float32 on the same batches."""
    sizes, B = [150, 97, 77], 64
    base, loss, shards, val = _mnist(sizes, torch.float32)
    pr, tr = _mnist_trainer(base, loss, shards, val, B, epochs=2)
    tr.run(tr.total)
    budgets = local_train.epoch_budgets(sizes, B, 2)
    r32 = _oracles(base, loss, shards, B)
    r64 = _oracles(base, loss, shards, B, dtype=torch.float64)
    for g in range(len(sizes)):
        r32[g].run(budgets[g]); r64[g].run(budgets[g])
        want = lto.flat(r64[g].model)
        e_fused = _rel(lto.flat(pr.models[g]).double(), want)
        e_torch = _rel(lto.flat(r32[g].model).double(), want)
        assert e_fused <= 4 * e_torch + 1e-6, (g, e_fused, e_torch)


# --------------------------------------------------------------------------------------- density ----
def _density(sizes, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    shards = [Shard(((torch.rand(m, 2, generator=g, dtype=torch.float64) - 0.5) * 1200).to(dtype),
                    (torch.rand(m, generator=g) < 0.3).to(dtype)) for m in sizes]
    val = Shard(((torch.rand(300, 2, generator=g, dtype=torch.float64) - 0.5) * 1200).to(dtype),
                (torch.rand(300, generator=g) < 0.3).to(dtype))
    torch.manual_seed(seed)
    return FourierNet([2, 256, 64, 64, 64, 1], scale=0.05, dtype=dtype), torch.nn.BCELoss(), shards, val


def _torch_density_vloss(model, val, vb):
    with torch.no_grad():
        out = torch.squeeze(model(val.x.to(DEV)))
        ps = torch.nn.functional.binary_cross_entropy(out, val.y.to(DEV), reduction="none")
    return sum_of_batch_means(ps, vb)


@pytest.mark.parametrize("opt", ["sgd", "adam", "adamw"])
def test_fp64_solo_density_matches_autograd(opt):
    sizes, B, lr = [700, 450, 130], 200, 1e-3
    base, loss, shards, val = _density(sizes, torch.float64)
    pr = local_train.build_problem("density", base, loss, shards, val, DEV, B, 100, SEED)
    budgets = local_train.epoch_budgets(sizes, B, 2)
    tr = local_train.LocalTrainer(pr, opt, lr, budgets)
    refs = _oracles(base, loss, shards, B, opt=opt, lr=lr, squeeze=True)
    tr.run(1)
    for g, r in enumerate(refs):
        r.run(1)
        assert _rel(lto.flat(pr.models[g]), lto.flat(r.model)) < 1e-9, g
    tr.run(tr.total - 1)
    assert tr.steps_taken() == budgets
    vl = pr._val_losses_local()
    for g, r in enumerate(refs):
        r.run(budgets[g] - 1)
        assert _rel(lto.flat(pr.models[g]), lto.flat(r.model)) < 1e-8, g
        assert vl[g].item() == pytest.approx(_torch_density_vloss(r.model, val, 100).item(), rel=1e-9)


def test_fp64_centralized_density_matches_autograd():
    sizes, B, lr, epochs = [700, 450, 130], 200, 1e-3, 3
    base, loss, shards, val = _density(sizes, torch.float64)
    union = Shard(torch.cat([s.x for s in shards]), torch.cat([s.y for s in shards]))
    hist = local_train.centralized(copy.deepcopy(base), loss, union, val, DEV, epochs, lr, B, 100, squeeze=True,
                                   verbose=False, seed=SEED)
    ref = _oracles(base, loss, [union], B, lr=lr, squeeze=True)[0]
    bpe = BatchSchedule(len(union), B).batches_per_epoch
    assert [h["epoch"] for h in hist] == list(range(epochs))
    for ep in range(epochs):
        ref.run(bpe)
        want = _torch_density_vloss(ref.model, val, 100).item()
        assert hist[ep]["top1_accuracy"] is None and isinstance(hist[ep]["validation_loss"], float)
        assert hist[ep]["validation_loss"] == pytest.approx(want, rel=1e-9), ep


def test_fp32_solo_density_within_bf16_tolerance():
    """bf16 tensor-core operands: the tolerance of tests/test_gpu_mlp.py for the first layer's gradient, on the change
    SGD made to the parameters (with Adam, coordinates whose gradient is round-off would step by +-lr either way)."""
    sizes, B, lr = [3000, 2000], 1000, 1e-2
    base, loss, shards, val = _density(sizes, torch.float32)
    pr = local_train.build_problem("density", base, loss, shards, val, DEV, B, 200, SEED)
    theta0 = [lto.flat(pr.models[g]).clone() for g in range(len(sizes))]
    budgets = local_train.epoch_budgets(sizes, B, 2)
    tr = local_train.LocalTrainer(pr, "sgd", lr, budgets)
    tr.run(tr.total)
    refs = _oracles(base, loss, shards, B, opt="sgd", lr=lr, squeeze=True)
    for g, r in enumerate(refs):
        r.run(budgets[g])
        want = lto.flat(r.model) - theta0[g]
        got = lto.flat(pr.models[g]) - theta0[g]
        assert _rel(got, want) < 0.12, g
    vf = pr._val_losses_local()
    for g, r in enumerate(refs):
        torch.testing.assert_close(vf[g], _torch_density_vloss(r.model, val, 200), rtol=5e-2, atol=5e-2)


# ------------------------------------------------------------------------------ determinism / graphs ----
def test_runs_are_bitwise_equal_and_graphs_equal_eager(monkeypatch):
    sizes, B = [150, 97, 77], 64
    base, loss, shards, val = _mnist(sizes, torch.float64)
    out = []
    for eager in (False, False, True):
        if eager:
            monkeypatch.setenv("NNDT_NO_GRAPH", "1")
        pr, tr = _mnist_trainer(base, loss, shards, val, B, epochs=2)
        assert tr.capturable == (not eager)
        tr.run(tr.total)
        torch.cuda.synchronize()
        out.append(pr.arena.theta.clone())
    assert torch.equal(out[0], out[1])
    assert torch.equal(out[0], out[2])


def test_online_density_runner_writes_solo_results(tmp_path):
    """``dist_online_dense_ex`` with ``train_solo: true, backend: fused``: the same keys, shapes, dtypes and CPU
    placement as the torch path."""
    from nn_distributed_training_b200.experiments import dist_online_dense_ex
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    data = str(tmp_path / "floor")
    write_dataset(data, n_paths=3, seed=0)
    with open("experiments/dist_online_dense_PAPER.yaml") as f:
        paper = yaml.safe_load(f)
    results = {}
    for backend in ("torch", "fused"):
        conf = copy.deepcopy(paper)
        e = conf["experiment"]
        e.update(output_metadir=str(tmp_path / backend))
        e["data"].update(data_dir=data, num_beams=8, beam_samps=10, collision_samps=20, spline_res=4,
                         num_validation_scans=20, border_width=8, num_scans_in_window=10, num_nodes=3)
        e["individual_training"].update(train_solo=True, train_batch_size=500, val_batch_size=500, epochs=2,
                                        verbose=False, backend=backend)
        conf["problem_configs"] = {"problem1": conf["problem_configs"]["problem1"]}
        pc = conf["problem_configs"]["problem1"]
        pc.update(train_batch_size=300, val_batch_size=400, comm_radius=300.0)
        pc["metrics"] = ["validation_loss"]
        pc["metrics_config"].update(evaluate_frequency=2)
        pc["optimizer_config"].update(outer_iterations=2, primal_iterations=1)
        path = tmp_path / f"{backend}.yaml"
        path.write_text(yaml.safe_dump(conf))
        dist_online_dense_ex.main(["x", str(path)])
        (run,) = os.listdir(tmp_path / backend)
        results[backend] = torch.load(tmp_path / backend / run / "solo_results.pt")
    t, f = results["torch"], results["fused"]
    assert sorted(t) == sorted(f) == [0, 1, 2]
    for g in t:
        assert sorted(t[g]) == sorted(f[g]) == ["mesh_grid", "mesh_grid_density", "validation_loss"]
        for key in t[g]:
            assert torch.is_tensor(f[g][key]) and f[g][key].device.type == "cpu", key
            assert f[g][key].shape == t[g][key].shape and f[g][key].dtype == t[g][key].dtype, key
        assert torch.equal(f[g]["mesh_grid"], t[g]["mesh_grid"])
        assert torch.isfinite(f[g]["validation_loss"]) and torch.isfinite(f[g]["mesh_grid_density"]).all()
