"""Multi-process worker for SPARQ-SGD (launched by torch.distributed.run from test_distributed_sparq.py): the cases of
``dist_worker.py``'s driver with ``alg_name: sparq_sgd`` on a fixed cycle whose edges cross ranks (no link drops: the
graph must not change), one and two local steps.  A node reads the trigger tails of its cross-rank neighbors and pulls a
code body only when its tail says so.  The rows compared exactly are theta and every declared row: x_hat, s, the
pending rows (code and tail) and the trigger counters."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "sparq_sgd": dw.Case([{"alg_name": "sparq_sgd", "alpha0": 0.05, "mu": 0.01, "gamma": 0.5, "compressor": "int8",
                           "threshold": 40.0},
                          {"alg_name": "sparq_sgd", "alpha0": 0.05, "mu": 0.01, "gamma": 0.5, "compressor": "sign",
                           "threshold": 40.0, "local_steps": 2}], link_drops=False),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
