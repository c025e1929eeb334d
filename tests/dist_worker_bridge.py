"""Multi-process worker for BRIDGE (launched by torch.distributed.run from test_distributed_bridge.py): the cases of
``dist_worker.py``'s driver with ``alg_name: bridge`` under either screen and attack, so the placement, the spin-delayed
loop with link drops and the sequence check, and the exact comparison against one process are the same as for the other
optimizers.  The attackers are the first and the last node (``dist_worker.VARIANTS['attack']``)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "bridge": dw.Case([{"alg_name": "bridge", "alpha0": 0.02, "mu": 0.001}],
                      variants={"screen": "trimmed_mean", "attack": "alie"}),
}
VARIANTS = {"screen": lambda v, N: {"screen": v, "b": 1} if v == "trimmed_mean" else {"screen": v}}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case and its flags from these tables
    dw.VARIANTS.update(VARIANTS)
    dw.main()
