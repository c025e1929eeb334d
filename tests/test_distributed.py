"""One rank per GPU (or per CPU process): the distributed run of every consensus optimizer must reproduce the
single-process run — gloo/world_size 2 here on CPU, NCCL + peer-mapped kernels on GPUs.  The cases are those of
``dist_worker.py``'s table."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "dist_worker.py")


def _launch(nproc, extra, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), WORKER] + extra
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)


def _cases(rows, port0):
    """``(case, graph, options)`` rows -> parameters ``(worker arguments, master port)`` with readable ids; every launch
    gets its own port."""
    out = []
    for i, (case, graph, opts) in enumerate(rows):
        args = ["--case", case, "--graph", graph] + [a for k, v in opts.items() for a in ("--" + k, str(v))]
        tags = [f"correction{v}" if k == "correction" else str(v) for k, v in opts.items() if k != "delayed"]
        name = "-".join([case, *tags, graph] + (["delayed"] if opts.get("delayed") else []))
        out.append(pytest.param(args, port0 + i, id=name))
    return out


TRIO = "dinno_dsgd_dsgt"

# The PyTorch path with two CPU ranks.  The directed cases gather in-neighbor rows (numerators, trackers) and the float64
# weights across ranks, each rank with its slice of the push-sum matrix; ``switching`` changes the directed graph every
# round.
GLOO_CASES = _cases([
    (TRIO, "cycle", {}), (TRIO, "wheel", {}),
    ("exact_diffusion", "wheel", {}),
    ("choco_sgd", "wheel", {}),
    ("sgp", "random_directed", {}), ("sgp", "switching", {}),
    ("push_diging", "random_directed", {}), ("push_diging", "switching", {}),
    ("dsgdm", "wheel", {"momentum": "local"}), ("dsgdm", "wheel", {"momentum": "quasi_global"}),
    ("beer", "wheel", {}),
    ("kgt", "wheel", {"correction": 1}), ("kgt", "wheel", {"correction": 0}),
    ("clipped_gossip", "cycle", {"clip": "none", "attack": "sign_flip"}),
    ("clipped_gossip", "wheel", {"clip": "adaptive", "attack": "sign_flip"}),
    ("clipped_gossip", "wheel", {"clip": "none", "attack": "alie"}),
    ("clipped_gossip", "cycle", {"clip": "adaptive", "attack": "alie"}),
], 29700)
GLOO_NODES = {"sgp": 6, "push_diging": 6}       # directed graphs of 6 nodes; 4 otherwise

# NCCL + peer-mapped consensus kernels, one rank per GPU.  ``pipeline`` (the trio): ``host`` pulls the rows from pinned
# host memory by the staging kernel inside multi-round graphs, peers announced by the first consensus kernel of each
# round; the single-process run uses resident shards.  ``delayed``: one rank is held back by spin kernels and every
# neighbor read is checked against its round tag; cases that allow a changing graph also drop links every round, which
# opens the write-after-read window of the double-buffered published rows.  On the directed cycle a rank reads only its
# predecessor, so without the wait for its readers it could run ahead of them and overwrite a buffer still being read;
# ``switching`` takes the readers from the previous round's graph.
NCCL_CASES = _cases([
    (TRIO, "cycle", {"pipeline": "auto"}), (TRIO, "complete", {"pipeline": "resident"}),
    (TRIO, "cycle", {"pipeline": "host"}), (TRIO, "wheel", {"delayed": 1}),
    ("exact_diffusion", "cycle", {"delayed": 0}), ("exact_diffusion", "complete", {"delayed": 0}),
    ("exact_diffusion", "wheel", {"delayed": 1}),
    ("choco_sgd", "cycle", {"delayed": 0}), ("choco_sgd", "complete", {"delayed": 0}),
    ("choco_sgd", "wheel", {"delayed": 1}),
    ("sgp", "directed_cycle", {"delayed": 0}), ("sgp", "exponential", {"delayed": 0}),
    ("sgp", "random_directed", {"delayed": 0}), ("sgp", "directed_cycle", {"delayed": 1}),
    ("sgp", "switching", {"delayed": 1}),
    ("push_diging", "directed_cycle", {"delayed": 0}), ("push_diging", "exponential", {"delayed": 0}),
    ("push_diging", "random_directed", {"delayed": 0}), ("push_diging", "directed_cycle", {"delayed": 1}),
    ("push_diging", "switching", {"delayed": 1}),
    ("dsgdm", "cycle", {"delayed": 0, "momentum": "local"}),
    ("dsgdm", "complete", {"delayed": 0, "momentum": "quasi_global"}),
    ("dsgdm", "wheel", {"delayed": 1, "momentum": "quasi_global"}),
    ("beer", "cycle", {"delayed": 0}), ("beer", "complete", {"delayed": 0}), ("beer", "wheel", {"delayed": 1}),
    ("kgt", "cycle", {"delayed": 0, "correction": 0}), ("kgt", "complete", {"delayed": 0, "correction": 1}),
    ("kgt", "wheel", {"delayed": 1, "correction": 1}),
    ("clipped_gossip", "cycle", {"delayed": 0, "clip": "none", "attack": "sign_flip"}),
    ("clipped_gossip", "complete", {"delayed": 0, "clip": "adaptive", "attack": "alie"}),
    ("clipped_gossip", "wheel", {"delayed": 1, "clip": "adaptive", "attack": "alie"}),
    ("clipped_gossip", "cycle", {"delayed": 1, "clip": "adaptive", "attack": "sign_flip"}),
], 29750)


@pytest.mark.parametrize("args,port", GLOO_CASES)
def test_gloo_two_ranks_match_single_process(args, port):
    nodes = GLOO_NODES.get(args[1], 4)
    r = _launch(2, ["--cuda", "0", "--nodes", str(nodes)] + args, port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("args,port", NCCL_CASES)
def test_nccl_peer_mapped_ranks_match_single_process(args, port):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    nproc = min(8, n)         # every GPU of the box: 2 on the development boxes, 8 on the scaling box
    r = _launch(nproc, ["--cuda", "1", "--nodes", str(3 * nproc)] + args, port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_gloo_online_density_runner_matches_single_process(tmp_path):
    """The YAML runner itself under torchrun (2 gloo ranks, 2 robots each): dynamic disk graph from gathered robot
    positions, planned topology tables, metrics gathered to rank 0 — same result files as the single-process run."""
    import glob

    import yaml
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    floor = str(tmp_path / "floor")
    write_dataset(floor, n_paths=4, seed=0)
    with open(os.path.join(ROOT, "experiments", "dist_online_dense_PAPER.yaml")) as f:
        base = yaml.safe_load(f)
    runner = os.path.join(ROOT, "experiments", "dist_online_dense_ex.py")
    outs = []
    for tag, nproc in (("single", 1), ("dist", 2)):
        conf = yaml.safe_load(yaml.safe_dump(base))
        e = conf["experiment"]
        out = str(tmp_path / tag)
        os.makedirs(out)
        e.update(output_metadir=out, use_cuda=False)
        e["data"].update(data_dir=floor, num_beams=8, beam_samps=10, collision_samps=20, spline_res=4,
                         num_validation_scans=20, border_width=8, num_scans_in_window=10, num_nodes=4)
        e["model"]["shape"] = [2, 32, 16, 1]
        e["individual_training"].update(train_solo=False)
        conf["problem_configs"] = {k: v for k, v in conf["problem_configs"].items() if v["optimizer_config"]["alg_name"] != "dsgd"}
        for pc in conf["problem_configs"].values():
            pc.update(train_batch_size=300, val_batch_size=400, comm_radius=300.0)
            pc["metrics_config"].update(evaluate_frequency=3)
            pc["optimizer_config"]["outer_iterations"] = 5
        cfg = os.path.join(out, "o.yaml")
        with open(cfg, "w") as f:
            yaml.safe_dump(conf, f)
        if nproc == 1:
            cmd = [sys.executable, runner, cfg]
        else:
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                   "--master-addr", "127.0.0.1", "--master-port", "29613", runner, cfg]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"),
                           cwd=os.path.join(ROOT, "experiments"))
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append(glob.glob(os.path.join(out, "*_dist_online_dense_PAPER"))[0])
    names = sorted(os.path.basename(p) for p in glob.glob(os.path.join(outs[0], "*_results.pt")))
    assert names and names == sorted(os.path.basename(p) for p in glob.glob(os.path.join(outs[1], "*_results.pt")))
    for n in names:
        a = torch.load(os.path.join(outs[0], n), weights_only=False)
        b = torch.load(os.path.join(outs[1], n), weights_only=False)
        va, vb = torch.stack(a["validation_loss"]), torch.stack(b["validation_loss"])
        assert va.shape == vb.shape and va.shape[1] == 4 and va.shape[0] >= 2
        assert torch.allclose(va, vb, rtol=1e-5, atol=1e-6)
        assert a["forward_pass_count"] == b["forward_pass_count"]


def test_gloo_mnist_paper_runner_matches_single_process(tmp_path):
    """dist_mnist_ex.py + dist_mnist_PAPER.yaml (hetero split, DiNNO / DSGT / DSGD) under torchrun with 2 gloo ranks:
    rank 0 writes the same files with the same metrics as the single-process run."""
    import glob

    import yaml
    with open(os.path.join(ROOT, "experiments", "dist_mnist_PAPER.yaml")) as f:
        base = yaml.safe_load(f)
    runner = os.path.join(ROOT, "experiments", "dist_mnist_ex.py")
    outs = []
    for tag, nproc in (("single", 1), ("dist", 2)):
        conf = yaml.safe_load(yaml.safe_dump(base))
        out = str(tmp_path / tag)
        os.makedirs(out)
        e = conf["experiment"]
        e.update(output_metadir=out, use_cuda=False, data_dir="/nonexistent")      # -> synthetic MNIST
        e["graph"].update(num_nodes=4)
        e["individual_training"].update(train_solo=False)
        for pc in conf["problem_configs"].values():
            pc["metrics_config"].update(evaluate_frequency=2)
            pc["optimizer_config"]["outer_iterations"] = 4
        cfg = os.path.join(out, "m.yaml")
        with open(cfg, "w") as f:
            yaml.safe_dump(conf, f)
        cmd = [sys.executable, runner, cfg] if nproc == 1 else \
            [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
             "--master-addr", "127.0.0.1", "--master-port", "29614", runner, cfg]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"),
                           cwd=os.path.join(ROOT, "experiments"))
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append(glob.glob(os.path.join(out, "*_dist_mnist_PAPER"))[0])
    files = [sorted(f for f in os.listdir(o) if not f.endswith(".yaml")) for o in outs]
    assert files[0] == files[1] == ["dinno_results.pt", "dsgd_results.pt", "dsgt_results.pt", "graph.gpickle"]
    for n in files[0][:3]:
        a = torch.load(os.path.join(outs[0], n), weights_only=False)
        b = torch.load(os.path.join(outs[1], n), weights_only=False)
        assert torch.allclose(torch.stack(a["top1_accuracy"]), torch.stack(b["top1_accuracy"]))
        assert torch.allclose(torch.stack(a["validation_loss"]), torch.stack(b["validation_loss"]), rtol=1e-5, atol=1e-7)
        assert a["forward_pass_count"] == b["forward_pass_count"]
