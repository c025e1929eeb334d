"""Multi-process worker for CHOCO-SGD and BEER with top-k codes (launched by torch.distributed.run from
test_distributed_topk.py): the cases of ``dist_worker.py`` with ``compressor: topk``, run by its driver, so the
placement, the spin-delayed loop and the exact comparison against one process are the same as for the other
compressors."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

CASES = {
    "choco_sgd_topk": dw.Case([{"alg_name": "choco_sgd", "alpha0": 0.05, "mu": 0.01, "gamma": 0.5,
                                "compressor": "topk", "topk_ratio": 0.01}], link_drops=False),
    "beer_topk": dw.Case([{"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "compressor": "topk",
                           "topk_ratio": 0.01}], link_drops=False),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from its table
    dw.main()
