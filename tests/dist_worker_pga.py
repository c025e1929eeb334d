"""Multi-process worker for Gossip-PGA (launched by torch.distributed.run from test_distributed_pga.py): the cases of
``dist_worker.py``'s driver with ``alg_name: gossip_pga`` on a cycle with link drops (they affect gossip rounds only).
Period 2 keeps global rounds two apart, so on a cycle of 3 nodes per rank the rank graph's diameter exceeds
``period - 1`` once there are four ranks or more; local SGD (``gossip: false``) pulls no row at all."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402


def torch_path(delayed, eng):
    """Exact on the PyTorch path, whose global mean adds the gathered rows in node order, as one process does; the
    fused global rounds add the ranks' fp64 partial sums in the reduction's order."""
    return eng is None


CASES = {
    "gossip_pga": dw.Case([{"alg_name": "gossip_pga", "alpha0": 0.05, "mu": 0.01, "period": 2},
                           {"alg_name": "gossip_pga", "alpha0": 0.05, "mu": 0.01, "period": 3, "gossip": False}],
                          exact=torch_path),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
