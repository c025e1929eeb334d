"""Multi-process worker for DP-DSGD / DECOR (launched by torch.distributed.run from test_distributed_dp.py): the cases
of ``dist_worker.py``'s driver with ``alg_name: dp_dsgd`` on a cycle whose edges cross ranks, with link drops in every
run (not only delayed ones), a clip that binds and pairwise noise: both ends of a cross-rank edge draw its noise on
their own.  The optimizer rows compared are theta; the ledger is checked against the single process's too."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker as dw  # noqa: E402

_make = dw.make


def make(ctx, case, graphs, conf, backend, delayed, pipeline):
    """``dist_worker.make`` with the delayed runs' link drops in every run."""
    return _make(ctx, case, graphs, conf, backend, True, pipeline)


_state_rows = dw.state_rows


def state_rows(pr, opt):
    """theta, plus the privacy ledger (every rank holds all N entries) as two ``[N, 1]`` rows."""
    import torch
    rows = _state_rows(pr, opt)
    rows["rho_eav"] = torch.as_tensor(opt.rho_eav).view(-1, 1)
    rows["rho_all"] = torch.as_tensor(opt.rho_all).view(-1, 1)
    return rows


CASES = {
    "dp_dsgd": dw.Case([{"alg_name": "dp_dsgd", "alpha0": 0.05, "mu": 0.01, "clip_norm": 0.5, "noise_multiplier": 0.01,
                         "pair_noise_multiplier": 0.02},
                        {"alg_name": "dp_dsgd", "alpha0": 0.05, "mu": 0.01, "clip_norm": 0.5, "noise_multiplier": 0.01}]),
}

if __name__ == "__main__":
    dw.CASES.update(CASES)      # this process only: the driver picks --case from this table
    dw.make = make
    dw.state_rows = state_rows
    dw.main()
