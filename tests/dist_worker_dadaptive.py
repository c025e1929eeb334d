"""Multi-process worker for decentralized AMSGrad / AdaGrad (launched by torch.distributed.run from
test_distributed_dadaptive.py): the cases of ``dist_worker.py``'s driver with ``alg_name: dadaptive``, with and without
the gossiped second moment, so the placement, the spin-delayed loop and the exact comparison against one process are
the same as for the other optimizers."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "dadaptive": dw.Case([{"alg_name": "dadaptive", "alpha": 0.002, "tracking": True}], exact=dw.unsummed,
                         variants={"variant": "amsgrad"}),
    "dadaptive_own": dw.Case([{"alg_name": "dadaptive", "alpha": 0.002, "tracking": False}], exact=dw.unsummed,
                             variants={"variant": "amsgrad"}),
}
VARIANTS = {"variant": lambda v, N: {"variant": v}}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case and its flags from these tables
    dw.VARIANTS.update(VARIANTS)
    dw.main()
