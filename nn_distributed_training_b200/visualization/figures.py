"""Static figures of the reference's notebooks, drawn with PIL so they work without matplotlib
(reference: floorplans/paperfig.ipynb + floorplans/lidar/lidar_example.ipynb -> ``lidar_figure``;
visualization/mnist_four.ipynb + online_density_vis.ipynb curves -> ``curves_figure`` / ``compare_runs_figure``;
visualization/online_density_vis.ipynb density panels -> ``density_panel``).

    python -m nn_distributed_training_b200.visualization.figures curves  <run_dir> out.png [--every 20]
    python -m nn_distributed_training_b200.visualization.figures compare out.png <run_dir> <run_dir> ... [--every 20]
    python -m nn_distributed_training_b200.visualization.figures density <run_dir> out.png [--node 0]
"""
from __future__ import annotations

import sys
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
from PIL import Image, ImageDraw

from .animations import _axes
from .results import _stack, density_image, load_results

ALG_COLORS = {"dinno": (255, 140, 0), "cadmm": (255, 140, 0), "dsgt": (50, 205, 50), "dsgd": (128, 0, 128),
              "exact_diffusion": (30, 144, 255), "choco_sgd": (220, 20, 60), "sgp": (0, 128, 128),
              "push_diging": (184, 134, 11), "dsgdm": (199, 21, 133), "beer": (0, 100, 0),
              "kgt": (70, 130, 180), "clipped_gossip": (139, 69, 19), "dadaptive": (106, 90, 205),
              "relaysum": (210, 105, 30), "bridge": (112, 128, 144),
              "powergossip": (0, 139, 139), "detag": (178, 34, 34),
              "gt_hsgd": (72, 61, 139), "gossip_pga": (218, 165, 32),
              "dp_dsgd": (199, 21, 133), "moniqua": (46, 139, 87), "cross_gradient": (0, 0, 205),
              "slowmo": (255, 99, 71)}
FALLBACK = [(31, 119, 180), (214, 39, 40), (44, 160, 44), (148, 103, 189), (140, 86, 75), (23, 190, 207)]


def _color(name: str, k: int):
    for key, col in ALG_COLORS.items():
        if name.lower().startswith(key):
            return col
    return FALLBACK[k % len(FALLBACK)]


def _consensus_to_mean(metrics) -> Optional[np.ndarray]:
    """``[evaluations, N]`` distance of every node to the mean of the normalised parameters."""
    ce = metrics.get("consensus_error")
    if not ce:
        return None
    rows = []
    for c in ce:
        d = c[1] if isinstance(c, tuple) else torch.as_tensor(c).mean(1)
        rows.append(np.asarray(torch.as_tensor(d).reshape(-1), dtype=np.float64))
    return np.stack(rows)


def _panel(size, series, title, every, log=False, band=True):
    """One axes box with mean curves (and min/max bands) of ``{name: [evaluations, N]}``."""
    vals = {k: (np.log10(np.maximum(v, 1e-12)) if log else v) for k, v in series.items() if v is not None and len(v)}
    if not vals:
        im, d, _ = _axes(size, (0, 1), (0, 1), title + " (no data)")
        return im
    tmax = max(v.shape[0] - 1 for v in vals.values()) * every
    lo = min(float(v.min()) for v in vals.values()); hi = max(float(v.max()) for v in vals.values())
    pad = 0.05 * max(hi - lo, 1e-9)
    im, d, px = _axes(size, (0, max(tmax, 1)), (lo - pad, hi + pad), title + (" (log10)" if log else ""))
    for k, (name, v) in enumerate(vals.items()):
        col = _color(name, k)
        v = v.reshape(v.shape[0], -1)
        t = np.arange(v.shape[0]) * every
        if band and v.shape[1] > 1 and v.shape[0] > 1:
            light = tuple(int(255 - 0.3 * (255 - c)) for c in col)
            d.polygon([px(x, y) for x, y in zip(t, v.max(1))] + [px(x, y) for x, y in zip(t[::-1], v.min(1)[::-1])], fill=light)
        if v.shape[0] > 1:
            d.line([px(x, y) for x, y in zip(t, v.mean(1))], fill=col, width=2)
        d.text((size[0] - 110, 28 + 13 * k), name[:16], fill=col)
    return im


def curves_figure(run_dir: str, out: str, evaluate_frequency: int = 20, size=(460, 320)) -> str:
    """Top-1 accuracy (or validation loss when there is no accuracy), validation loss and consensus error of every
    problem of a run: the three panels of ``results.plot_run``."""
    res = load_results(run_dir)
    acc = {n: _stack(m.get("top1_accuracy")) for n, m in res.items()}
    vl = {n: _stack(m.get("validation_loss")) for n, m in res.items()}
    ce = {n: _consensus_to_mean(m) for n, m in res.items()}
    panels = []
    if any(v is not None for v in acc.values()):
        panels.append(_panel(size, acc, "top-1 accuracy (mean, min-max)", evaluate_frequency))
    panels.append(_panel(size, vl, "validation loss", evaluate_frequency, log=True))
    panels.append(_panel(size, ce, "consensus error (distance to mean)", evaluate_frequency, log=True, band=False))
    fig = Image.new("RGB", (size[0] * len(panels), size[1]), (255, 255, 255))
    for i, p in enumerate(panels):
        fig.paste(p, (i * size[0], 0))
    fig.save(out)
    return out


def compare_runs_figure(run_dirs: Sequence[str], out: str, evaluate_frequency: int = 20, titles: Optional[Sequence[str]] = None,
                        key: str = "top1_accuracy", size=(420, 320)) -> str:
    """One panel per run directory (e.g. complete / cycle / random graphs side by side, visualization/mnist_four.ipynb)."""
    panels = []
    for i, rd in enumerate(run_dirs):
        res = load_results(rd)
        series = {n: _stack(m.get(key)) for n, m in res.items()}
        panels.append(_panel(size, series, titles[i] if titles else rd.rstrip("/").split("/")[-1][-40:], evaluate_frequency,
                             log=key != "top1_accuracy"))
    fig = Image.new("RGB", (size[0] * len(panels), size[1]), (255, 255, 255))
    for i, p in enumerate(panels):
        fig.paste(p, (i * size[0], 0))
    fig.save(out)
    return out


def _grey(a: np.ndarray, scale: int = 1) -> Image.Image:
    im = Image.fromarray((255 * (1.0 - np.clip(a, 0.0, 1.0))).astype(np.uint8), mode="L")
    if scale != 1:
        im = im.resize((max(1, int(im.width * scale)), max(1, int(im.height * scale))), Image.NEAREST)
    return im.convert("RGB")


def density_panel(metrics_by_name: Dict[str, dict], out: str, lidar=None, node: int = 0, index: int = -1, height: int = 240) -> str:
    """Ground truth (when the lidar is given) next to the occupancy map learned by ``node`` under every algorithm
    (visualization/online_density_vis.ipynb: odense_allalg_mesh)."""
    tiles, labels = [], []
    if lidar is not None:
        tiles.append(_grey(np.asarray(lidar.img, dtype=np.float64)))           # img is [ny, nx]: rows are y
        labels.append("Ground Truth")
    for name, m in metrics_by_name.items():
        if m.get("mesh_grid_density"):
            tiles.append(_grey(density_image(m, node=node, index=index)))
            labels.append(name)
    if not tiles:
        raise ValueError("no mesh_grid_density metric in the given results")
    tiles = [t.resize((max(1, int(t.width * height / t.height)), height), Image.NEAREST) for t in tiles]
    fig = Image.new("RGB", (sum(t.width for t in tiles) + 6 * (len(tiles) - 1), height + 18), (255, 255, 255))
    d = ImageDraw.Draw(fig)
    x = 0
    for t, lab in zip(tiles, labels):
        fig.paste(t, (x, 18))
        d.text((x + 4, 3), lab, fill=(0, 0, 0))
        x += t.width + 6
    fig.save(out)
    return out


def lidar_figure(lidar, datasets: Sequence, out: str, highlight: int = 0, max_points: int = 20000, scale: float = 0.5) -> str:
    """Floor plan with the robots' trajectories and the scan samples of one robot: free-space samples dark blue,
    occupied samples gold (floorplans/paperfig.ipynb, lidar_example.ipynb).  ``datasets`` are lidar datasets exposing
    ``scan_locs [T, 2]`` and their samples as a ``Shard`` (``x [P, 2]``, ``y [P]``)."""
    img = np.asarray(lidar.img, dtype=np.float64)
    W, H = int(lidar.nx), int(lidar.ny)
    base = _grey(img).resize((max(1, int(W * scale)), max(1, int(H * scale))), Image.BILINEAR)
    d = ImageDraw.Draw(base)

    def px(p):            # world coordinates are centred pixels: x in [-nx/2, nx/2], y in [-ny/2, ny/2]
        return ((float(p[0]) + W / 2) * scale, (float(p[1]) + H / 2) * scale)
    for k, ds in enumerate(datasets):
        locs = np.asarray(ds.scan_locs)
        col = (255, 69, 0) if k == highlight else FALLBACK[k % len(FALLBACK)]
        if len(locs) > 1:
            d.line([px(p) for p in locs], fill=col, width=3 if k == highlight else 1)
    ds = datasets[highlight]
    x = np.asarray(ds.shard.x.cpu(), dtype=np.float64)[:max_points]
    y = np.asarray(ds.shard.y.cpu(), dtype=np.float64).reshape(-1)[:max_points]
    for p, v in zip(x, y):
        cx, cy = px(p)
        if v >= 1.0:
            d.ellipse([cx - 2, cy - 2, cx + 2, cy + 2], fill=(255, 215, 0))
        else:
            d.point((cx, cy), fill=(0, 0, 139))
    base.save(out)
    return out


def _arg(argv, flag, default):
    return type(default)(argv[argv.index(flag) + 1]) if flag in argv else default


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    kind = argv[0]
    every = _arg(argv, "--every", 20)
    if kind == "curves":
        return curves_figure(argv[1], argv[2], every)
    if kind == "compare":
        dirs = [a for i, a in enumerate(argv[2:]) if not a.startswith("--") and argv[2:][i - 1] != "--every"]
        return compare_runs_figure(dirs, argv[1], every)
    if kind == "density":
        return density_panel(load_results(argv[1]), argv[2], node=_arg(argv, "--node", 0))
    raise SystemExit(f"unknown figure '{kind}'")


if __name__ == "__main__":
    print(main())
