"""Push-DIGing with one rank per GPU (or per CPU process) on directed graphs: the distributed run must reproduce the
single-process run — gloo with two ranks on the CPU, NCCL + peer-mapped consensus kernels on GPUs."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "dist_worker_push_diging.py")


def _launch(nproc, extra, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), WORKER] + extra
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)


@pytest.mark.parametrize("graph,port", [("random_directed", 29651), ("switching", 29652)])
def test_gloo_two_ranks_match_single_process(graph, port):
    """The PyTorch path: in-neighbor numerators, trackers and the float64 weights gathered across ranks, each rank's
    slice of the push-sum matrix; ``switching`` changes the directed graph every round."""
    r = _launch(2, ["--cuda", "0", "--nodes", "6", "--graph", graph], port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("graph,delayed,port", [("directed_cycle", 0, 29653), ("exponential", 0, 29654),
                                                ("random_directed", 0, 29655), ("directed_cycle", 1, 29656),
                                                ("switching", 1, 29657)])
def test_nccl_peer_mapped_ranks_match_single_process(graph, delayed, port):
    """``delayed``: one rank is held back by spin kernels and every in-neighbor read is checked against its round tag.
    On the directed cycle a rank reads only its predecessor, so without the wait for its readers it could run ahead of
    them and overwrite a buffer still being read; ``switching`` takes the readers from the previous round's graph.  The
    result must equal the single-process run exactly."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    nproc = min(8, n)
    r = _launch(nproc, ["--cuda", "1", "--nodes", str(3 * nproc), "--graph", graph, "--delayed", str(delayed)], port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
