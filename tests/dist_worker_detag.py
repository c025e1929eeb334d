"""Multi-process worker for DeTAG (launched by torch.distributed.run from test_distributed_detag.py): the cases of
``dist_worker.py``'s driver with ``alg_name: detag`` on a cycle, without link drops (DeTAG needs a fixed graph).  The
driver compares theta and every ``STATE`` row (``y``, ``g_old`` and the published ``z``) with one process exactly.  On
the cycle split across ranks every gossip sub-step crosses ranks, so a round makes ``gossip_steps`` announcements."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "detag": dw.Case([{"alg_name": "detag", "alpha": 0.02, "gossip_steps": 3, "accelerate": True},
                      {"alg_name": "detag", "alpha": 0.02, "gossip_steps": 2, "accelerate": False}],
                     link_drops=False),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.main()
