"""Multi-process worker for GT-HSGD (launched by torch.distributed.run from test_distributed_gt_hsgd.py): the cases of
``dist_worker.py``'s driver with ``alg_name: gt_hsgd`` on a cycle with link drops (the tracking invariant holds for any
doubly stochastic W).  The driver compares theta and every ``STATE`` row (``y``, ``v`` and ``theta_prev``) with one
process exactly."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "gt_hsgd": dw.Case([{"alg_name": "gt_hsgd", "alpha": 0.02, "beta": 0.3},
                        {"alg_name": "gt_hsgd", "alpha": 0.02, "beta": 1.0}]),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
