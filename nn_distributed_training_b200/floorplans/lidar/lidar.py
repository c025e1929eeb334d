"""Simulated 2-D lidar over a floor-plan density image, and the datasets built on it
(reference: floorplans/lidar/lidar.py — ``Lidar2D`` :9, ``ClippedLidar2D`` :139,
``RandomPoseLidarDataset`` :240, ``TrajectoryLidarDataset`` :290,
``OnlineTrajectoryLidarDataset`` :336, ``interpolate_waypoints`` :427).

The reference casts every beam of every scan in nested Python loops (minutes for the paper's
~2 400 scans x 20 beams per robot).  Here ``scan_batch`` marches *all* beams of *all* poses at
once with array ops (coarse march -> fine search -> power-law resampling), producing the same
points scan for scan; ``scan(pos)`` is the single-pose view of it.  Datasets keep their points
as one ``Shard`` (dense tensors) so the problems can place them in HBM, and the online
sliding-window logic is index arithmetic over a draw counter (``data.sampler.OnlineWindowSchedule``)
instead of a popped Python list.
"""
from __future__ import annotations

import numpy as np
import scipy.interpolate as interp
import torch
from PIL import Image

from ...data.sampler import OnlineWindowSchedule
from ...data.shards import Shard


def _load_density_image(img, border_width):
    if isinstance(img, (str, bytes)) or hasattr(img, "__fspath__"):
        arr = np.asarray(Image.open(img)).astype(float) / 255.0
    else:
        arr = np.array(img, dtype=float)
    if arr.ndim == 3:
        arr = arr[..., 0]
    if border_width != 0:
        # same slices as the reference (:38-42): the last row/column stay untouched
        arr[:, :border_width] = 1.0
        arr[:border_width, :] = 1.0
        arr[:, -border_width:-1] = 1.0
        arr[-border_width:-1, :] = 1.0
    return arr


class _LidarBase:
    beam_stop_thresh = 0.5

    def _setup_grid(self, img, border_width, beam_length):
        self.img = _load_density_image(img, border_width)
        self.nx = self.img.shape[1]
        self.ny = self.img.shape[0]
        self.beam_len = beam_length * max(self.nx, self.ny)
        # world axes are centred pixels
        self.xs = self.nx * np.linspace(-0.5, 0.5, num=self.nx)
        self.ys = self.ny * np.linspace(-0.5, 0.5, num=self.ny)
        self.density = interp.RectBivariateSpline(self.xs, self.ys, self.img.T)

    def _check_free(self, pos):
        d = self.density.ev(pos[:, 0], pos[:, 1])
        if (d >= self.beam_stop_thresh).any():
            bad = pos[np.argmax(d >= self.beam_stop_thresh)]
            print(bad)
            raise NameError("Cannot lidar scan from point with high density.")

    def _beam_vectors(self):
        angs = np.linspace(-np.pi, np.pi, num=self.num_beams, endpoint=False)
        return self.beam_len * np.stack([np.cos(angs), np.sin(angs)], axis=1)  # [Bm, 2]

    def scan(self, pos):
        """Scan from one pose ``pos`` of shape (1, 2): rows ``(x, y, density)``."""
        return self.scan_batch(np.asarray(pos, dtype=float).reshape(1, 2))[0]


class Lidar2D(_LidarBase):
    """Queryable 2-D lidar: coarse march, fine collision search, weighted beam samples."""

    def __init__(self, img_dir, num_beams, beam_length, beam_samps, samp_distribution_factor,
                 collision_samps, fine_samps, border_width=0):
        self.num_beams = num_beams
        self.beam_samps = beam_samps
        self.collision_samps = collision_samps
        self.fine_samps = fine_samps
        self.samp_df = samp_distribution_factor
        self._setup_grid(img_dir, border_width, beam_length)

    def _spline_tables(self, device):
        """Knots / coefficients of the fitted bicubic spline on ``device`` (for ops/csrc/lidar.cu)."""
        key = str(device)
        if getattr(self, "_tables", None) is None or self._tables[0] != key:
            tx, ty = self.density.get_knots()
            c = self.density.get_coeffs()
            t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=device)
            self._tables = (key, t(tx), t(ty), t(c))
        return self._tables[1:]

    def cuda_args(self, device):
        """Spline tables and beam parameters of ops/csrc/lidar.cu's ``lidar_scan`` / ``lidar_density``, without the
        poses and the output."""
        tx, ty, c = self._spline_tables(device)
        return dict(tx=tx.data_ptr(), ty=ty.data_ptr(), coef=c.data_ptr(), ntx=tx.numel(), nty=ty.numel(),
                    num_beams=self.num_beams, beam_samps=self.beam_samps, collision_samps=self.collision_samps,
                    fine_samps=self.fine_samps, beam_len=float(self.beam_len), samp_df=float(self.samp_df))

    def scan_batch_cuda(self, pos, device="cuda"):
        """GPU twin of ``scan_batch`` (one thread per pose x beam; fp64)."""
        from ...ops import load_ext
        ext = load_ext(required=True)
        pos = np.asarray(pos, dtype=float).reshape(-1, 2)
        self._check_free(pos)
        poses = torch.as_tensor(pos, dtype=torch.float64, device=device).contiguous()
        out = torch.empty(pos.shape[0], self.num_beams * self.beam_samps, 3, dtype=torch.float64, device=device)
        ext.lidar_scan(dict(self.cuda_args(device), poses=poses.data_ptr(), n_poses=pos.shape[0], out=out.data_ptr()))
        return out

    def scan_batch(self, pos, chunk=512, device=None):
        """All beams of all poses ``pos [P,2]`` -> ``[P, num_beams*beam_samps, 3]``.  With a CUDA
        ``device`` the scans are generated by the GPU kernel and returned as a NumPy array."""
        device = device if device is not None else getattr(self, "scan_device", None)
        if device is not None and torch.device(device).type == "cuda":
            return self.scan_batch_cuda(pos, device).cpu().numpy()
        pos = np.asarray(pos, dtype=float).reshape(-1, 2)
        self._check_free(pos)
        out = np.empty((pos.shape[0], self.num_beams * self.beam_samps, 3))
        for a in range(0, pos.shape[0], chunk):
            out[a: a + chunk] = self._scan_chunk(pos[a: a + chunk])
        return out

    def _scan_chunk(self, pos):
        P, Bm, S = pos.shape[0], self.num_beams, self.beam_samps
        thr = self.beam_stop_thresh
        bv = self._beam_vectors()                                        # [Bm,2]
        tc = np.linspace(0.0, 1.0, num=self.collision_samps)              # [C]
        coarse = pos[:, None, None, :] + tc[None, None, :, None] * bv[None, :, None, :]   # [P,Bm,C,2]
        cvals = self.density.ev(coarse[..., 0].ravel(), coarse[..., 1].ravel()).reshape(P, Bm, -1)
        hit = np.argmax(cvals >= thr, axis=2)                             # 0 == no collision
        has_hit = hit > 0
        pi, bi = np.nonzero(has_hit)
        # beam end point: full beam, or the refined collision point
        end = pos[:, None, :] + bv[None, :, :]                            # [P,Bm,2]
        t_beam = np.broadcast_to(np.linspace(0.0, 1.0, S), (P, Bm, S)).copy()
        if pi.size:
            hi = hit[pi, bi]
            coll = coarse[pi, bi, hi]
            last_empty = coarse[pi, bi, hi - 1]
            tf = np.linspace(0.0, 1.0, self.fine_samps)
            fine = last_empty[:, None, :] + tf[None, :, None] * (coll - last_empty)[:, None, :]
            fvals = self.density.ev(fine[..., 0].ravel(), fine[..., 1].ravel()).reshape(pi.size, -1)
            fhit = np.argmax(fvals >= thr, axis=1)
            end[pi, bi] = fine[np.arange(pi.size), fhit]
            t_beam[pi, bi] = np.power(np.linspace(0.0, 1.0, S), self.samp_df)
        pnts = pos[:, None, None, :] + t_beam[..., None] * (end - pos[:, None, :])[:, :, None, :]   # [P,Bm,S,2]
        vals = self.density.ev(pnts[..., 0].ravel(), pnts[..., 1].ravel()).reshape(P, Bm, S, 1)
        return np.concatenate([pnts, vals], axis=3).reshape(P, Bm * S, 3)


class ClippedLidar2D(_LidarBase):
    """Coarse-only variant: a beam is cut right after its first colliding sample, so scans
    have a variable number of points (reference :139-237)."""

    def __init__(self, img_dir, num_beams, beam_length, beam_samps, border_width=0):
        self.num_beams = num_beams
        self.beam_samps = beam_samps
        self._setup_grid(img_dir, border_width, beam_length)

    def scan_batch(self, pos):
        pos = np.asarray(pos, dtype=float).reshape(-1, 2)
        self._check_free(pos)
        P, Bm, S = pos.shape[0], self.num_beams, self.beam_samps
        bv = self._beam_vectors()
        t = np.linspace(0.0, 1.0, num=S)
        pnts = pos[:, None, None, :] + t[None, None, :, None] * bv[None, :, None, :]
        vals = self.density.ev(pnts[..., 0].ravel(), pnts[..., 1].ravel()).reshape(P, Bm, S)
        hit = np.argmax(vals >= self.beam_stop_thresh, axis=2)
        keep = (np.arange(S)[None, None, :] <= hit[..., None]) | (hit[..., None] == 0)
        full = np.concatenate([pnts, vals[..., None]], axis=3)
        return [full[p][keep[p]] for p in range(P)]

    def scan(self, pos):
        return self.scan_batch(np.asarray(pos, dtype=float).reshape(1, 2))[0]


def interpolate_waypoints(x, y, spline_res):
    """Cubic interpolation of a waypoint polyline to ``spline_res*(len-1)`` poses (:427-435)."""
    i = np.arange(len(x))
    ii = np.linspace(0, i.max(), spline_res * i.max())
    xi = interp.interp1d(i, x, kind="cubic")(ii)
    yi = interp.interp1d(i, y, kind="cubic")(ii)
    return np.hstack((xi.reshape(-1, 1), yi.reshape(-1, 1)))


class _LidarDataset(torch.utils.data.Dataset):
    """Points of a list of scans as dense tensors: ``scans [M,3]``, ``shard`` = (xy, label)."""

    def _finish(self, scan_list, round_density):
        self.scans = torch.from_numpy(np.vstack(scan_list))
        if round_density:
            self.scans[:, 2] = torch.round(self.scans[:, 2])
        self.shard = Shard(self.scans[:, :2].contiguous(), self.scans[:, 2].contiguous())
        self.tds = torch.utils.data.TensorDataset(self.shard.x, self.shard.y)

    def __getitem__(self, idx):
        return self.tds[idx]

    def __len__(self):
        return len(self.tds)


class RandomPoseLidarDataset(_LidarDataset):
    """``num_scans`` scans from uniformly sampled free-space poses (:240-287)."""

    def __init__(self, lidar, num_scans, round_density=True):
        super().__init__()
        self.lidar = lidar
        c, locs = 0, []
        while c < num_scans:
            xs = np.random.choice(lidar.xs, num_scans)
            ys = np.random.choice(lidar.ys, num_scans)
            free = lidar.density.ev(xs, ys) < 0.5
            c += int(free.sum())
            locs.append(np.stack([xs[free], ys[free]], axis=1))
        self.scan_locs = np.vstack(locs)[:num_scans, :]
        self._finish(list(lidar.scan_batch(self.scan_locs)), round_density)


def _trajectory_poses(lidar, waypoints, spline_res):
    traj = interpolate_waypoints(waypoints[:, 0], waypoints[:, 1], spline_res)
    # normalised [-1,1]^2 waypoints -> centred pixel coordinates
    return traj * np.array([lidar.nx * 0.5, lidar.ny * 0.5]).reshape(1, 2)


class TrajectoryLidarDataset(_LidarDataset):
    """Scans along a cubic path through normalised waypoints (:290-333)."""

    def __init__(self, lidar, waypoints, spline_res, round_density=True):
        super().__init__()
        self.lidar = lidar
        self.scan_locs = _trajectory_poses(lidar, waypoints, spline_res)
        self._finish(list(lidar.scan_batch(self.scan_locs)), round_density)


class OnlineTrajectoryLidarDataset(_LidarDataset):
    """Trajectory dataset consumed through a sliding window of ``num_scans_in_window`` scans
    (:336-424).  ``curr_pos`` is the robot pose of the current window; draws are served from
    a keyed permutation of the window and advance it when exhausted."""

    def __init__(self, lidar, waypoints, spline_res, num_scans_in_window, round_density=True, seed=0, node=0):
        super().__init__()
        self.lidar = lidar
        self.scan_locs = _trajectory_poses(lidar, waypoints, spline_res)
        self.num_scans = self.scan_locs.shape[0]
        self._finish(list(lidar.scan_batch(self.scan_locs)), round_density)
        self.num_scans_in_window = num_scans_in_window
        self.scan_size = lidar.num_beams * lidar.beam_samps
        self.schedule = OnlineWindowSchedule(self.num_scans, self.scan_size, num_scans_in_window)
        self.seed, self.node = seed, node
        self.draws = 0

    def reset_cursor(self):
        """Restart the stream (each problem config starts from the first window — SURVEY Q14)."""
        self.draws = 0

    @property
    def curr_scan_idx(self):
        return self.schedule.scan_cursor_at(self.draws)

    @property
    def curr_pos(self):
        return self.scan_locs[self.curr_scan_idx, :]

    def pos_after(self, draws: int):
        return self.scan_locs[self.schedule.scan_cursor_at(draws), :]

    def next_indices(self, count: int, device="cpu") -> torch.Tensor:
        idx = self.schedule.indices(self.draws, count, self.seed, self.node, device=device)
        self.draws += count
        return idx

    def __getitem__(self, index):
        # DataLoader protocol: the requested index is ignored, the stream decides (:385-392)
        return self.tds[int(self.next_indices(1)[0])]
