"""Multi-process worker for RelaySum (launched by torch.distributed.run from test_distributed_relaysum.py): the cases of
``dist_worker.py``'s driver with ``alg_name: relaysum`` on a path (``--graph path``), without link drops (RelaySum
needs a fixed tree), so the placement, the spin-delayed loop and the exact comparison against one process are the same
as for the other optimizers."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "relaysum": dw.Case([{"alg_name": "relaysum", "alpha0": 0.05, "mu": 0.01}], link_drops=False),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
