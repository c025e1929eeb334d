"""SlowMo across ranks: the distributed run reproduces the single-process run, bit for bit on two gloo CPU ranks and to
round-off on NCCL, whose global rounds reduce the fp64 partial sums over NVLS (with a delayed rank too), with cycle edges
that cross ranks.  The cases are those of ``dist_worker_slowmo.py``: over gossip at period 2, and over local SGD with
Nesterov base momentum at period 3."""
import os
import subprocess
import sys

import pytest
import torch

from test_distributed import _cases

WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_worker_slowmo.py")


def _launch(nproc, extra, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), WORKER] + extra
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="2"))


GLOO_CASES = _cases([("slowmo", "cycle", {})], 30140)

NCCL_CASES = _cases([
    ("slowmo", "cycle", {"delayed": 0}),
    ("slowmo", "cycle", {"delayed": 1}),
], 30150)


@pytest.mark.parametrize("args,port", GLOO_CASES)
def test_gloo_two_ranks_match_single_process(args, port):
    r = _launch(2, ["--cuda", "0", "--nodes", "4"] + args, port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("args,port", NCCL_CASES)
def test_nccl_peer_mapped_ranks_match_single_process(args, port):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    nproc = min(8, n)
    r = _launch(nproc, ["--cuda", "1", "--nodes", str(3 * nproc)] + args, port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
