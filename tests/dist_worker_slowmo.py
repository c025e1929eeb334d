"""Multi-process worker for SlowMo (launched by torch.distributed.run from test_distributed_slowmo.py): the cases of
``dist_worker.py``'s driver with ``alg_name: slowmo`` on a cycle with link drops (they affect gossip rounds only), over
gossip at period 2 and over local SGD with base momentum at period 3.  The outer update adds no traffic: a global round
exchanges what Gossip-PGA's does."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402


def torch_path(delayed, eng):
    """Exact on the PyTorch path, whose global mean adds the gathered rows in node order, as one process does; the
    fused global rounds add the ranks' fp64 partial sums in the reduction's order."""
    return eng is None


CASES = {
    "slowmo": dw.Case([{"alg_name": "slowmo", "alpha0": 0.05, "mu": 0.01, "period": 2, "slow_momentum": 0.5},
                       {"alg_name": "slowmo", "alpha0": 0.05, "mu": 0.01, "period": 3, "gossip": False,
                        "slow_momentum": 0.7, "slow_lr": 1.5, "base_momentum": 0.9, "nesterov": True}],
                      exact=torch_path),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
