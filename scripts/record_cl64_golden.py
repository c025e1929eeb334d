"""Records the float64 cluster kernel's gradient-slot digests and loss partials at every configuration of
tests/test_gpu_mnist_cl64_push.py into tests/golden/cl64_grads.npz (run on an H100 from the kernel whose outputs are
to be kept).

    python scripts/record_cl64_golden.py [--out tests/golden/cl64_grads.npz]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_gpu_mnist_cl64_push as t  # noqa: E402

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=t.GOLDEN)
    args = ap.parse_args()
    out = {}
    for cfg in t.CONFIGS:
        os.environ["NNDT_TC_SPLIT"] = str(cfg[0])
        loss, dig, _ = t.run(*cfg)
        out[t.key(*cfg) + "_loss"], out[t.key(*cfg) + "_digest"] = loss, dig
        print(t.key(*cfg), loss.shape, dig.shape, flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez_compressed(args.out, **out)
    print("wrote", args.out)
