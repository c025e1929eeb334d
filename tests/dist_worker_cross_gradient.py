"""Multi-process worker for cross-gradient gossip (launched by torch.distributed.run from
test_distributed_cross_gradient.py): the cases of ``dist_worker.py``'s driver with ``alg_name: cross_gradient`` on a
fixed cycle (the cross-gradients travel back over the edges of one graph, so no link drops).  The driver compares theta
with one process exactly; the cross-gradients cross ranks as per-slot rows, RelaySum's way."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "cross_gradient": dw.Case([{"alg_name": "cross_gradient", "alpha0": 0.05, "mu": 0.01, "cross_weight": 1.0},
                               {"alg_name": "cross_gradient", "alpha0": 0.05, "cross_weight": 0.3}],
                              link_drops=False),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
