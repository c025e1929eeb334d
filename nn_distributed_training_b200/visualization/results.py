"""Result inspection and figures (reference: visualization/*.ipynb, centralized/*.ipynb —
notebooks that consume ``<problem>_results.pt`` / ``graph.gpickle`` and define the de-facto
output-file contract, SURVEY Appendix B).

Everything here works on the files the runners write.  Numbers (final accuracy / loss,
rounds-to-threshold as in ``visualization/scaling_plots.ipynb``) are computed without any
plotting dependency; figures are produced when matplotlib is available.

    python -m nn_distributed_training_b200.visualization.results <run_dir> [--plot out.svg]
"""
from __future__ import annotations

import glob
import os
import sys
from typing import Dict, List, Optional

import numpy as np
import torch

from ..experiments.common import read_gpickle


def load_results(run_dir: str) -> Dict[str, dict]:
    """``{problem_name: metrics dict}`` for every ``*_results.pt`` in a run directory."""
    out = {}
    for f in sorted(glob.glob(os.path.join(run_dir, "*_results.pt"))):
        name = os.path.basename(f)[: -len("_results.pt")]
        if name != "solo":
            out[name] = torch.load(f, map_location="cpu", weights_only=False)
    return out


def _stack(metric_list) -> Optional[np.ndarray]:
    if not metric_list:
        return None
    return np.stack([np.asarray(torch.as_tensor(m).cpu()) for m in metric_list])


def summarize_run(run_dir: str, eval_every: Optional[int] = None) -> Dict[str, dict]:
    res = load_results(run_dir)
    summary = {}
    for name, m in res.items():
        s = {}
        # a run with Byzantine nodes is summarised over its honest nodes
        byz = set(m.get("byzantine_nodes", ()))
        acc = _stack(m.get("top1_accuracy"))
        if acc is not None:
            a = acc[-1][[i for i in range(acc.shape[1]) if i not in byz]]
            s["final_top1_mean"] = float(a.mean()); s["final_top1_min"] = float(a.min())
        vl = _stack(m.get("validation_loss"))
        if vl is not None:
            honest = [i for i in range(vl.shape[1]) if i not in byz]
            s["final_val_loss_mean"] = float(vl[-1][honest].mean()); s["first_val_loss_mean"] = float(vl[0][honest].mean())
        ce = m.get("consensus_error")
        if ce:
            last = ce[-1]
            d = last[1] if isinstance(last, tuple) else torch.as_tensor(last).mean(1)
            s["final_consensus_max"] = float(torch.as_tensor(d).max())
        if m.get("forward_pass_count"):
            s["forward_passes"] = int(m["forward_pass_count"][-1])
        summary[name] = s
        print(name, s)
    g = os.path.join(run_dir, "graph.gpickle")
    if os.path.exists(g):
        graph = read_gpickle(g)
        print("graph:", graph.number_of_nodes(), "nodes,", graph.number_of_edges(), "edges")
    return summary


def rounds_to_threshold(metrics: dict, threshold: float, evaluate_frequency: int, key="top1_accuracy") -> Optional[int]:
    """First evaluated round whose node-mean metric reaches ``threshold`` (the quantity plotted in
    visualization/scaling.svg: rounds to 50/90/97 % mean top-1)."""
    vals = _stack(metrics.get(key))
    if vals is None:
        return None
    mean = vals.reshape(vals.shape[0], -1).mean(1)
    hit = np.nonzero(mean >= threshold)[0]
    return int(hit[0] * evaluate_frequency) if hit.size else None


def plot_run(run_dir: str, out: str, evaluate_frequency: int = 20):
    try:
        import matplotlib
        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
    except ImportError:
        from .figures import curves_figure          # same three panels drawn with PIL
        summarize_run(run_dir)
        return curves_figure(run_dir, out[:-4] + ".png" if out.endswith(".svg") else out, evaluate_frequency)
    res = load_results(run_dir)
    fig, axes = plt.subplots(1, 3, figsize=(14, 4))
    for name, m in res.items():
        acc, vl = _stack(m.get("top1_accuracy")), _stack(m.get("validation_loss"))
        x = None
        if acc is not None:
            x = np.arange(acc.shape[0]) * evaluate_frequency
            axes[0].plot(x, acc.mean(1), label=name)
            axes[0].fill_between(x, acc.min(1), acc.max(1), alpha=0.2)
        if vl is not None:
            x = np.arange(vl.shape[0]) * evaluate_frequency
            axes[1].semilogy(x, vl.mean(1), label=name)
        ce = m.get("consensus_error")
        if ce:
            d = np.asarray([float(torch.as_tensor(c[1] if isinstance(c, tuple) else torch.as_tensor(c).mean(1)).max()) for c in ce])
            axes[2].semilogy(np.arange(len(d)) * evaluate_frequency, d, label=name)
    for ax, t in zip(axes, ("top-1 accuracy (mean, min-max band)", "validation loss", "consensus error (max distance to mean)")):
        ax.set_title(t); ax.set_xlabel("communication round"); ax.legend()
    fig.tight_layout(); fig.savefig(out)
    return out


def density_image(metrics: dict, node: int = 0, index: int = -1):
    """Reshape a ``mesh_grid_density`` entry into the 2-D image it samples (every 8th pixel)."""
    mesh = torch.as_tensor(metrics["mesh_inputs"])
    dens = torch.as_tensor(metrics["mesh_grid_density"][index])[node].reshape(-1)
    xs, ys = torch.unique(mesh[:, 0]), torch.unique(mesh[:, 1])
    return dens.reshape(len(ys), len(xs)).numpy()


if __name__ == "__main__":
    run = sys.argv[1]
    if "--plot" in sys.argv:
        plot_run(run, sys.argv[sys.argv.index("--plot") + 1])
    else:
        summarize_run(run)
