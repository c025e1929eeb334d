"""Multi-process worker for PowerGossip (launched by torch.distributed.run from test_distributed_powergossip.py): the
cases of ``dist_worker.py``'s driver with ``alg_name: powergossip`` on a cycle, without link drops (PowerGossip needs a
fixed graph).  The driver compares theta and every ``STATE`` row (the vectors ``vec`` and the messages ``msg``) with
one process exactly; on the cycle some edges cross ranks, so an endpoint whose vectors drifted from its peer's would
differ from the single-process run, where ``test_powergossip.py`` checks both endpoints bit for bit."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "powergossip": dw.Case([{"alg_name": "powergossip", "alpha0": 0.05, "mu": 0.01, "gamma": 0.8}], link_drops=False),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
