"""ClippedGossip with one rank per GPU (or per CPU process), Byzantine nodes on the first and the last rank: the
distributed run must reproduce the single-process run — gloo with two ranks on the CPU, NCCL + peer-mapped consensus
kernels on GPUs."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "dist_worker_clipped_gossip.py")


def _launch(nproc, extra, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), WORKER] + extra
    env = dict(os.environ, OMP_NUM_THREADS="2")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)


@pytest.mark.parametrize("clip,attack,graph,port", [("none", "sign_flip", "cycle", 29691),
                                                    ("adaptive", "sign_flip", "wheel", 29692),
                                                    ("none", "alie", "wheel", 29693),
                                                    ("adaptive", "alie", "cycle", 29694)])
def test_gloo_two_ranks_match_single_process(clip, attack, graph, port):
    r = _launch(2, ["--cuda", "0", "--nodes", "4", "--graph", graph, "--clip", clip, "--attack", attack], port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("graph,delayed,clip,attack,port", [("cycle", 0, "none", "sign_flip", 29695),
                                                            ("complete", 0, "adaptive", "alie", 29696),
                                                            ("wheel", 1, "adaptive", "alie", 29697),
                                                            ("cycle", 1, "adaptive", "sign_flip", 29698)])
def test_nccl_peer_mapped_ranks_match_single_process(graph, delayed, clip, attack, port):
    """``delayed``: link drops change the graph every round, one rank is held back by spin kernels and every neighbor
    read at round start is checked against its round tag; the result must equal the single-process run exactly."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    nproc = min(8, n)
    r = _launch(nproc, ["--cuda", "1", "--nodes", str(3 * nproc), "--graph", graph, "--delayed", str(delayed),
                        "--clip", clip, "--attack", attack], port)
    assert "DIST_RESULT PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
