"""Multi-process worker for Moniqua (launched by torch.distributed.run from test_distributed_moniqua.py): the cases of
``dist_worker.py``'s driver with ``alg_name: moniqua`` on both bases, on a cycle whose edges cross ranks, with link drops
in every run (not only delayed ones): a node decodes the code rows of its cross-rank neighbors against its own theta.
The rows compared exactly are theta and every declared row: the pending codes, the margin counters and (Exact
Diffusion base) psi."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

_make = dw.make


def make(ctx, case, graphs, conf, backend, delayed, pipeline):
    """``dist_worker.make`` with the delayed runs' link drops in every run."""
    return _make(ctx, case, graphs, conf, backend, True, pipeline)


CASES = {
    "moniqua": dw.Case([{"alg_name": "moniqua", "alpha0": 0.05, "mu": 0.01, "bits": 4, "theta_bound": 0.3},
                        {"alg_name": "moniqua", "alpha0": 0.05, "mu": 0.01, "bits": 8, "theta_bound": 0.3,
                         "base": "exact_diffusion"}]),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.make = make
    dw.main()
