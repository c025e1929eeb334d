"""GPU numerics: fused sm_90a kernels vs plain PyTorch fp32 references."""
import copy

import networkx as nx
import numpy as np
import pytest
import torch

import kernel_oracles as ko
from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.data.sampler import BatchSchedule
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.optimizers import DiNNO, DSGD, DSGT
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
METRICS = ["forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"]


@pytest.fixture(scope="module", autouse=True)
def _fp32_references():
    """The fp32 autograd comparisons in this module mean fp32, not TF32."""
    with ko.fp32_references():
        yield


def _problem(N, B, backend, opt_conf, M=300, float_inputs=False, seed=0, graph=None, eval_every=1000):
    torch.manual_seed(seed)
    data = synthetic_mnist(M * N, seed=3)
    val = synthetic_mnist(200, seed=4)
    shards = [data.select(torch.arange(i * M, (i + 1) * M)) for i in range(N)]
    if float_inputs:
        from nn_distributed_training_b200.data.shards import Shard
        shards = [Shard(s.inputs(torch.arange(len(s)), torch.float32), s.y) for s in shards]
        val = Shard(val.inputs(torch.arange(len(val)), torch.float32), val.y)
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": METRICS,
            "metrics_config": {"evaluate_frequency": eval_every}, "optimizer_config": opt_conf}
    return DistMNISTProblem(graph or nx.cycle_graph(N), MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(),
                            shards, val, DEV, conf, backend=backend, seed=7)


def _assert_grads_close(a, b):
    """fp32 summation order differs from ATen's, so a ReLU / max-pool unit whose
    pre-activation is ~1e-7 can land on the other side of 0 and flip one sample's
    contribution to one row; allow <1% such coordinates but bound the global error."""
    bad = (a - b).abs() > 2e-5 + 2e-3 * b.abs()
    assert bad.float().mean().item() < 0.01
    rel = (a - b).norm() / b.norm().clamp_min(1e-12)
    assert rel.item() < 2e-2, rel.item()


def _assert_mostly_close(a, b, frac=0.1, rel=1e-2):
    """Adam's m/(sqrt(v)+eps) amplifies 1e-7 rounding differences on coordinates whose loss
    gradient is ~0 (dead units); require all but a sliver of coordinates to agree tightly and
    the whole state to agree in norm."""
    bad = (a - b).abs() > 2e-5 + 2e-3 * b.abs()
    assert bad.float().mean().item() < frac, bad.float().mean().item()
    assert ((a - b).norm() / b.norm().clamp_min(1e-12)).item() < rel


def test_extension_loaded():
    from nn_distributed_training_b200.ops import load_ext
    assert load_ext(required=True) is not None


@pytest.mark.parametrize("m,B", [(300, 64), (64, 64), (1000, 37), (5, 8)])
def test_device_sampler_matches_python(m, B):
    from nn_distributed_training_b200.ops import load_ext
    ext = load_ext(required=True)
    out = torch.zeros(B, dtype=torch.int32, device=DEV)
    size = torch.zeros(1, dtype=torch.int32, device=DEV)
    sched = BatchSchedule(m, B)
    for call in [0, 1, 4, 17, 123]:
        ext.debug_batch_indices(m, B, call, 7, 5, out.data_ptr(), size.data_ptr())
        ref = sched.indices(call, 7, 5)
        n = int(size.item())
        assert n == len(ref)
        assert out[:n].cpu().tolist() == ref.tolist()


@pytest.mark.parametrize("B,float_inputs", [(64, False), (24, False), (64, True), (100, False)])
def test_fwdbwd_matches_autograd(B, float_inputs):
    conf = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}
    fused = _problem(3, B, "fused", conf, M=150, float_inputs=float_inputs)
    ref = _problem(3, B, "torch", conf, M=150, float_inputs=float_inputs)
    assert fused.backend == "fused" and ref.backend == "torch"
    ref.arena.theta.copy_(fused.arena.theta)
    for step in range(4):  # crosses an epoch boundary (partial batch) when B does not divide 150
        lf = fused.compute_grads().clone()
        lr = ref.compute_grads().clone()
        torch.testing.assert_close(lf, lr, rtol=2e-4, atol=2e-5)
        _assert_grads_close(fused.arena.grad, ref.arena.grad)
    assert fused.forward_cnt == ref.forward_cnt
    assert (fused.calls == ref.calls).all()


def test_eval_matches_torch():
    conf = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}
    fused = _problem(3, 64, "fused", conf)
    ref = _problem(3, 64, "torch", conf)
    ref.arena.theta.copy_(fused.arena.theta)
    pf, of = fused._validate_local()
    prf, orf = ref._validate_local()
    torch.testing.assert_close(pf, prf, rtol=2e-4, atol=2e-5)
    assert (of != orf).float().mean().item() < 0.01
    fused.evaluate_metrics()
    ref.evaluate_metrics()
    torch.testing.assert_close(fused.metrics["validation_loss"][0], ref.metrics["validation_loss"][0],
                               rtol=1e-4, atol=1e-6)


DINNO = {"alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.01, "outer_iterations": 7,
         "primal_iterations": 2, "primal_optimizer": "adam", "persistant_primal_opt": False,
         "primal_lr_start": 0.005, "primal_lr_finish": 0.0005, "lr_decay_type": "log", "profile": False}
DSGD_C = {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.01, "outer_iterations": 7, "profile": False}
DSGT_C = {"alg_name": "dsgt", "alpha": 0.02, "init_grads": True, "outer_iterations": 7, "profile": False}


@pytest.mark.parametrize("cls,conf", [(DiNNO, DINNO), (DiNNO, dict(DINNO, primal_optimizer="sgd")),
                                      (DiNNO, dict(DINNO, primal_optimizer="adamw", persistant_primal_opt=True)),
                                      (DSGD, DSGD_C), (DSGT, DSGT_C), (DSGT, dict(DSGT_C, init_grads=False))])
@pytest.mark.parametrize("graph", ["cycle", "wheel", "complete"])
def test_fused_training_matches_torch_ops(cls, conf, graph):
    """Whole fused round programs (CUDA graph replay) vs the PyTorch consensus ops driving
    the same fused forward/backward, 7 rounds, fp32."""
    N = 5
    G = {"cycle": nx.cycle_graph(N), "wheel": nx.wheel_graph(N), "complete": nx.complete_graph(N)}[graph]
    a = _problem(N, 32, "fused", conf, graph=G, eval_every=3)
    b = _problem(N, 32, "fused", conf, graph=G, eval_every=3)
    b.arena.theta.copy_(a.arena.theta)
    oa = cls(a, DEV, copy.deepcopy(conf))
    ob = cls(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    oa.train()
    ob.train()
    assert oa._program.eng.sum_mode == (graph == "complete")     # complete graph -> network-sum kernels
    _assert_mostly_close(a.arena.theta, b.arena.theta)
    assert a.forward_cnt == b.forward_cnt
    assert len(a.metrics["validation_loss"]) == len(b.metrics["validation_loss"]) == 3
    if cls is DSGT:
        _assert_mostly_close(oa.y, ob.y)


def test_consensus_kernels_fp64_with_autograd_model():
    """fp64 arena on the GPU: autograd forward/backward + fused fp64 consensus kernels (eager)."""
    torch.manual_seed(0)
    N, B = 4, 16
    g = torch.Generator().manual_seed(0)
    train = [torch.utils.data.TensorDataset(torch.randn(B, 1, 28, 28, generator=g, dtype=torch.float64),
                                            torch.randint(0, 10, (B,), generator=g)) for _ in range(N)]
    val = torch.utils.data.TensorDataset(torch.randn(32, 1, 28, 28, generator=g, dtype=torch.float64),
                                         torch.randint(0, 10, (32,), generator=g))
    outs = []
    for backend in ("auto", "torch"):
        conf = dict(DINNO, consensus_backend=backend)
        pconf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 16, "metrics": METRICS,
                 "metrics_config": {"evaluate_frequency": 100}, "optimizer_config": conf}
        torch.manual_seed(1)
        pr = DistMNISTProblem(nx.wheel_graph(N), MNISTConvNet(3, 5, 64, dtype=torch.float64), torch.nn.NLLLoss(),
                              train, val, DEV, pconf, backend="torch")   # autograd model (float64 has fused kernels too now)
        assert pr.backend == "torch"
        DiNNO(pr, DEV, conf).train()
        outs.append(pr.arena.theta.clone())
    bad = (outs[0] - outs[1]).abs() > 1e-8 + 1e-6 * outs[1].abs()
    assert bad.double().mean().item() < 1e-3


@pytest.mark.parametrize("mode", ["gpu_pull", "staged"])
def test_host_fed_pipeline_matches_resident(mode):
    """Host-fed rounds (inputs cross PCIe every round) and staged-resident rounds (same staging kernel, HBM source)
    must train exactly like the resident pipeline: all draw the same rows from the same stateless sampler."""
    outs = []
    for pipeline in ("resident", "staged" if mode == "staged" else "host"):
        conf = dict(DINNO, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)   # 100/32: partial batches + epoch wrap
        pr.conf["input_pipeline"] = pipeline
        opt = DiNNO(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        outs.append((pr.arena.theta.clone(), pr.forward_cnt, pr.calls.copy()))
        if pipeline == "host":
            assert torch.isfinite(pr.fused.loss_host).all() and pr.fused.loss_host.abs().sum() > 0
    torch.testing.assert_close(outs[0][0], outs[1][0], rtol=0, atol=0)
    assert outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()


@pytest.mark.parametrize("pipeline", ["staged", "host"])
def test_dsgt_init_grads_with_host_fed_and_staged_pipelines(pipeline):
    """The paper's DSGT config (init_grads: true) through the host-fed / staged input pipelines: the one initial
    gradient draw runs on the resident shards, the stream takes over at the next draw — identical to the resident run."""
    outs = []
    for pl in ("resident", pipeline):
        conf = dict(DSGT_C, outer_iterations=12)
        pr = _problem(4, 32, "fused", conf, M=100, eval_every=1000)
        pr.conf["input_pipeline"] = pl
        opt = DSGT(pr, DEV, conf)
        opt.run_rounds(5)
        opt.run_rounds(4)
        torch.cuda.synchronize()
        assert opt._program.pipeline == pl
        outs.append((pr.arena.theta.clone(), pr.forward_cnt, pr.calls.copy()))
    torch.testing.assert_close(outs[0][0], outs[1][0], rtol=0, atol=0)
    assert outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()


def test_fused_consensus_metric_matches_torch():
    """The fused metric kernel (used at evaluation points of fused runs) vs the torch normalize/cdist oracle."""
    from nn_distributed_training_b200.ops import consensus_ref
    conf = dict(DINNO, outer_iterations=6)
    pr = _problem(5, 32, "fused", conf, graph=nx.wheel_graph(5), eval_every=2)
    DiNNO(pr, DEV, conf).train()
    d_all, d_mean = pr.metrics["consensus_error"][-2]          # evaluated before round 4 with the fused kernel
    assert d_all.shape == (5, 5) and d_mean.shape == (5, 1)
    # recompute the last evaluation point's value from the final parameters for a sanity range, and an exact check now
    eng, kfn = pr._metric_engine
    a, m = eng.consensus_metric(kfn())
    ra, rm = consensus_ref.consensus_error(pr.all_theta().double())
    torch.testing.assert_close(a, ra.cpu(), rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(m, rm.cpu(), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("cls,conf", [(DiNNO, dict(DINNO, persistant_primal_opt=True, outer_iterations=6)),
                                      (DSGD, dict(DSGD_C, outer_iterations=6)), (DSGT, dict(DSGT_C, outer_iterations=6))])
def test_fused_checkpoint_resume_is_bit_exact(tmp_path, cls, conf):
    """Crash after an ODD round (the published rows of the resumed round live in parity 1), resume in a fresh
    problem/optimizer on the fused path: parameters equal the uninterrupted run bit for bit."""
    from nn_distributed_training_b200.parallel.context import DistContext
    from nn_distributed_training_b200.utils import checkpoint as ckpt
    full = _problem(4, 32, "fused", conf, M=100)
    cls(full, DEV, copy.deepcopy(conf)).train()
    first = _problem(4, 32, "fused", conf, M=100)
    o1 = cls(first, DEV, copy.deepcopy(conf))
    ckpt.attach(o1, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)))
    o1.oits = 3                      # "crash" after round 3
    o1.train()
    assert o1.k == 3
    second = _problem(4, 32, "fused", conf, M=100)
    o2 = cls(second, DEV, copy.deepcopy(conf))
    ckpt.attach(o2, str(tmp_path), "run", every=3, ctx=DistContext.single(torch.device(DEV)), resume=True)
    assert o2.k == 3
    o2.train()
    assert torch.equal(second.arena.theta, full.arena.theta)
    assert second.forward_cnt == full.forward_cnt


@pytest.mark.parametrize("cls,conf", [(DiNNO, DINNO), (DSGT, DSGT_C)])
def test_sequence_check_passes_and_detects_stale_rows(cls, conf):
    """``debug_sequence_check``: every published row is tagged with its round and every neighbor read verifies the
    tag (SURVEY 5.2).  A clean run raises nothing; a corrupted tag is reported by ``engine.check()``."""
    c = dict(copy.deepcopy(conf), debug_sequence_check=True)
    pr = _problem(5, 32, "fused", c, graph=nx.wheel_graph(5))
    opt = cls(pr, DEV, c)
    opt.run_rounds(4)
    torch.cuda.synchronize()
    eng = opt._program.eng
    eng.check()
    assert int(eng.seq_buf.local[opt.k & 1].min()) == opt.k       # rows of the next round to be read are tagged k
    eng.seq_buf.local[opt.k & 1, 2] = 12345                        # node 2's row now claims a different round
    opt.run_rounds(1)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="sequence check"):
        eng.check()


@pytest.mark.parametrize("cls,conf", [(DiNNO, DINNO), (DSGD, DSGD_C), (DSGT, dict(DSGT_C, init_grads=False))])
def test_fused_link_drop_fault_injection_matches_torch_ops(cls, conf):
    """Time-varying graphs on the fused path: the link drops of ``fault_injection`` become per-round topology tables
    (several graphs, isolated nodes included) that the kernels index by the device round counter; the PyTorch
    consensus ops walking the same graph sequence are the oracle."""
    outs = []
    for backend in ("fused", "torch"):
        pr = _problem(6, 32, "fused", conf, graph=nx.cycle_graph(6), eval_every=1000)
        pr.conf["fault_injection"] = {"link_drop_prob": 0.5, "seed": 3, "from_round": 1, "to_round": 6}
        pr._init_faults()
        opt = cls(pr, DEV, dict(copy.deepcopy(conf), consensus_backend="auto" if backend == "fused" else "torch"))
        opt.train()
        outs.append(pr.arena.theta.clone())
        if backend == "fused":
            assert len(opt._program.eng.topos) > 2            # several distinct faulted graphs were tabulated
            opt._program.eng.check()
    _assert_mostly_close(outs[0], outs[1])


# ---- generic conv-net kernel (csrc/mnist_generic.cu): every MNISTConvNet shape, fp32 and fp64 ---------------------
def _generic_problem(shape, dtype, backend, B=32, N=3, M=150, eval_every=1000, conf=None):
    torch.manual_seed(0)
    data = synthetic_mnist(M * N, seed=3)
    val = synthetic_mnist(200, seed=4)
    shards = [data.select(torch.arange(i * M, (i + 1) * M)) for i in range(N)]
    conf = conf or {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}
    pconf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": METRICS,
             "metrics_config": {"evaluate_frequency": eval_every}, "optimizer_config": conf}
    model = MNISTConvNet(*shape)
    if dtype == torch.float64:
        model = model.double()
    return DistMNISTProblem(nx.cycle_graph(N), model, torch.nn.NLLLoss(), shards, val, DEV, pconf, backend=backend, seed=7)


@pytest.mark.parametrize("shape,dtype,B", [((3, 5, 64), torch.float64, 64), ((3, 5, 64), torch.float64, 37),
                                           ((8, 3, 128), torch.float64, 32), ((8, 3, 128), torch.float32, 32),
                                           ((2, 5, 32), torch.float32, 24), ((4, 3, 64), torch.float64, 16),
                                           ((6, 5, 128), torch.float32, 64)])
def test_generic_convnet_kernel_matches_autograd(shape, dtype, B):
    fused = _generic_problem(shape, dtype, "fused", B=B)
    ref = _generic_problem(shape, dtype, "torch", B=B)
    assert fused.backend == "fused" and fused.fused.generic and ref.backend == "torch"
    ref.arena.theta.copy_(fused.arena.theta)
    for step in range(4):
        lf = fused.compute_grads().clone()
        lr = ref.compute_grads().clone()
        if dtype == torch.float64:
            torch.testing.assert_close(lf, lr, rtol=1e-6, atol=1e-7)      # loss partials are stored as float
            torch.testing.assert_close(fused.arena.grad, ref.arena.grad, rtol=1e-9, atol=1e-11)
        else:
            torch.testing.assert_close(lf, lr, rtol=2e-4, atol=2e-5)
            _assert_grads_close(fused.arena.grad, ref.arena.grad)
    pf, of = fused._validate_local()
    prf, orf = ref._validate_local()
    if dtype == torch.float64:
        torch.testing.assert_close(pf, prf, rtol=1e-9, atol=1e-11)
        assert (of == orf).all()
    else:
        torch.testing.assert_close(pf, prf, rtol=2e-4, atol=2e-5)


def test_generic_kernel_env_switch_on_paper_shape_fp32(monkeypatch):
    """NNDT_MNIST_GENERIC=1 routes the paper shape through the generic kernel too (A/B switch); same gradients."""
    monkeypatch.setenv("NNDT_MNIST_GENERIC", "1")
    fused = _generic_problem((3, 5, 64), torch.float32, "fused", B=64)
    monkeypatch.delenv("NNDT_MNIST_GENERIC")
    spec = _generic_problem((3, 5, 64), torch.float32, "fused", B=64)
    assert fused.fused.generic and not spec.fused.generic
    spec.arena.theta.copy_(fused.arena.theta)
    fused.compute_grads(); spec.compute_grads()
    _assert_grads_close(fused.arena.grad, spec.arena.grad)


@pytest.mark.parametrize("cls,conf", [(DiNNO, DINNO), (DSGD, DSGD_C), (DSGT, DSGT_C)])
def test_fp64_fused_training_matches_torch_fp64(cls, conf):
    """The float64 arm (bench headline): fused fp64 forward/backward + fp64 consensus kernels under CUDA graphs against
    autograd + the PyTorch consensus ops in float64 — agreement to fp64 round-off, not fp32."""
    a = _generic_problem((3, 5, 64), torch.float64, "fused", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b = _generic_problem((3, 5, 64), torch.float64, "torch", B=32, N=5, eval_every=3, conf=copy.deepcopy(conf))
    b.arena.theta.copy_(a.arena.theta)
    oa = cls(a, DEV, copy.deepcopy(conf))
    ob = cls(b, DEV, dict(copy.deepcopy(conf), consensus_backend="torch"))
    oa.train()
    ob.train()
    rel = ((a.arena.theta - b.arena.theta).norm() / b.arena.theta.norm()).item()
    assert rel < 1e-8, rel
    assert a.forward_cnt == b.forward_cnt


# ---- K-split cluster kernel (csrc/mnist_tc.cu) ------------------------------------------------------------
@pytest.mark.parametrize("B,float_inputs", [(64, False), (37, False), (64, True), (8, False)])
def test_tc_kernel_matches_batch_split_kernel_and_autograd(B, float_inputs, monkeypatch):
    """The tensor-core kernel (default for the paper shape at batch <= 64) against the mma.sync batch-split kernel
    (NNDT_MNIST_TC=0) and against PyTorch autograd: 3xTF32 keeps fp32-level agreement."""
    conf = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}
    monkeypatch.setenv("NNDT_MNIST_TC", "1")
    tc = _problem(3, B, "fused", conf, M=150, float_inputs=float_inputs)
    monkeypatch.setenv("NNDT_MNIST_TC", "0")
    old = _problem(3, B, "fused", conf, M=150, float_inputs=float_inputs)
    monkeypatch.delenv("NNDT_MNIST_TC")
    ref = _problem(3, B, "torch", conf, M=150, float_inputs=float_inputs)
    assert tc.fused.tc and tc.fused.S in (1, 2, 4) and not old.fused.tc
    old.arena.theta.copy_(tc.arena.theta)
    ref.arena.theta.copy_(tc.arena.theta)
    for step in range(4):
        lt = tc.compute_grads().clone()
        lo = old.compute_grads().clone()
        lr = ref.compute_grads().clone()
        torch.testing.assert_close(lt, lr, rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(lt, lo, rtol=2e-4, atol=2e-5)
        _assert_grads_close(tc.arena.grad, ref.arena.grad)
        _assert_grads_close(tc.arena.grad, old.arena.grad)
    assert (tc.calls == ref.calls).all()


@pytest.mark.parametrize("B", [64, 37, 8])
def test_fp64_cluster_kernel_matches_generic_kernel_and_autograd(B, monkeypatch):
    """csrc/mnist_cl64.cu (K-split cluster kernel, the float64 arm of the paper shape) against the batch-split generic
    fp64 kernel (NNDT_MNIST_CL64=0) and PyTorch autograd in float64."""
    cl = _generic_problem((3, 5, 64), torch.float64, "fused", B=B)
    monkeypatch.setenv("NNDT_MNIST_CL64", "0")
    gen = _generic_problem((3, 5, 64), torch.float64, "fused", B=B)
    monkeypatch.delenv("NNDT_MNIST_CL64")
    ref = _generic_problem((3, 5, 64), torch.float64, "torch", B=B)
    assert cl.fused.cl64 and not gen.fused.cl64
    gen.arena.theta.copy_(cl.arena.theta)
    ref.arena.theta.copy_(cl.arena.theta)
    for step in range(4):
        lc, lg, lr = cl.compute_grads().clone(), gen.compute_grads().clone(), ref.compute_grads().clone()
        torch.testing.assert_close(lc, lr, rtol=1e-6, atol=1e-7)
        torch.testing.assert_close(cl.arena.grad, ref.arena.grad, rtol=1e-9, atol=1e-11)
        torch.testing.assert_close(cl.arena.grad, gen.arena.grad, rtol=1e-9, atol=1e-11)
    assert (cl.calls == ref.calls).all()


# ---- the cluster kernels at every instantiation the selector launches, against fp64 oracles ---------------------
def _bench_layout_problem(L, B, dtype):
    """bench.py's data layout at L nodes: one class per node, uint8 rows normalised in-kernel, a cycle, the paper's
    net.  A node's shard holds B + B // 2 + 1 rows, so its second draw is a partial batch and its third opens epoch 1."""
    M = B + B // 2 + 1
    shards = [synthetic_mnist(M, seed=100 + g, classes=[g % 10]) for g in range(L)]
    conf = {"problem_name": "t", "train_batch_size": B, "val_batch_size": 64, "metrics": METRICS,
            "metrics_config": {"evaluate_frequency": 1000},
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.001, "outer_iterations": 2, "profile": False}}
    torch.manual_seed(0)
    base = MNISTConvNet(3, 5, 64, dtype=dtype)
    pr = DistMNISTProblem(nx.cycle_graph(L), base, torch.nn.NLLLoss(), shards, synthetic_mnist(64, seed=1), DEV, conf,
                          backend="fused", seed=7)
    for l in range(L):                      # a different network per node, so a node mix-up cannot go unnoticed
        pr.arena.theta[l] *= 1.0 + 0.03 * l
    return pr


@pytest.mark.parametrize("nsplit,L", [(4, 3), (2, 10), (1, 12)])
@pytest.mark.parametrize("B", [64, 37, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cluster_kernels_match_fp64_oracle_at_every_instantiation(dtype, B, nsplit, L):
    """mnist_tc_train_kernel<MS> (fp32) and mnist_cl64_train_kernel<MS> (fp64) at MS = 16, 32, 64 samples per cluster:
    the batch splits per node the selector picks on a 132-SM H100 for 3, 10 (bench.py) and 12 nodes.  The oracle is
    float64 autograd on the rows the kernel drew.  fp64: agreement to 1e-9.  fp32 (3xTF32): the error is at most 0.1x
    that of a 1xTF32 emulation of the three fc1-sized contractions, per tensor and per 16 x 8 block."""
    if torch.cuda.get_device_properties(DEV).multi_processor_count != 132:
        pytest.skip("node counts chosen for the 132 SMs of an H100 SXM")
    pr = _bench_layout_problem(L, B, dtype)
    fz, spec = pr.fused, pr.base_model.spec
    assert (fz.cl64 if dtype == torch.float64 else fz.tc) and fz.S == nsplit
    assert f"_train_kernel<{64 // nsplit}>" in fz.kernel_name
    mean, std = pr.shards.norm
    worst = {}
    for step in range(3):                   # full batch, partial batch, first batch of the next epoch
        calls = pr.calls.copy()
        loss = fz.compute_grads().clone()
        for l in range(L):
            rows = ko.batch_rows(pr.shards.sizes, B, pr.seed, l, int(calls[l]), pr.placement.lo).to(DEV)
            x, y, th = pr.shards.x[rows], pr.shards.y[rows], pr.arena.theta[l]
            lr, gr = ko.convnet_fp64(th, spec, x, y, mean, std)
            if dtype == torch.float64:
                torch.testing.assert_close(loss[l], lr, rtol=1e-6, atol=1e-7)       # loss partials are stored as float
                torch.testing.assert_close(pr.arena.grad[l], gr, rtol=1e-9, atol=1e-11)
                continue
            gt = ko.convnet_fp64(th, spec, x, y, mean, std, tf32_fc1=True)[1]
            assert abs(loss[l].item() - lr.item()) <= 1e-5 * abs(lr.item()), (l, step, loss[l].item(), lr.item())
            rat = ko.assert_close_to_oracle(pr.arena.grad[l].double(), gr, gt, ko.CONVNET_FRAC, spec=spec)
            for k, v in rat.items():
                worst[k] = max(worst.get(k, 0.0), *v)
    if worst:
        print(f"\nRATIO mnist_tc<{64 // nsplit}> B={B}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))
