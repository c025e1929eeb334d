"""ops/csrc/lidar.cu against float64 oracles: the bicubic spline density (``lidar_density``) against scipy's FITPACK
evaluation, and the batched scans (``lidar_scan``) against the reference's recorded scans and the NumPy twin
``Lidar2D._scan_chunk``, at every branch of the beam march: no hit, a hit at the first coarse sample (the last empty
point is the pose itself), beams leaving the image (the spline clamped at its end knots), every power-law exponent,
beam counts that do not fill a thread block, and the smallest sample counts.

Every scan case is first checked to be well posed: the smallest |density - 0.5| over its coarse and fine samples
(from the oracle) must exceed 1e-9, so a one-ulp difference in cos, sin or an FMA cannot flip a hit index and the
1e-9 bound holds for the right reason."""
import copy
import functools
import os

import numpy as np
import pytest
import torch

from nn_distributed_training_b200.floorplans.lidar import Lidar2D, interpolate_waypoints
from nn_distributed_training_b200.ops import load_ext

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAN = os.path.join(ROOT, "floorplans", "32_data", "floor_img.png")
PATH = os.path.join(ROOT, "floorplans", "32_data", "tight_paths", "1.npy")
THR = Lidar2D.beam_stop_thresh


@functools.lru_cache(maxsize=None)
def _paper_lidar():
    """dist_online_dense_PAPER's lidar on the reference floor plan (1608 x 2167 pixels)."""
    return Lidar2D(PLAN, 20, 0.2, 25, 1.0, 50, 3, border_width=30)


def _variant(base, beam_length=None, **kw):
    """``base`` with other beam parameters and the same fitted spline."""
    v = copy.copy(base)
    for k, val in kw.items():
        setattr(v, k, val)
    if beam_length is not None:
        v.beam_len = beam_length * max(v.nx, v.ny)
    return v


def _trajectory(lidar, spline_res=30):
    wp = np.load(PATH)
    return interpolate_waypoints(wp[:, 0], wp[:, 1], spline_res) * np.array([lidar.nx * 0.5, lidar.ny * 0.5])


# ---- the spline ---------------------------------------------------------------------------------------------------
def _density_gpu(lidar, xy):
    ext = load_ext(required=True)
    n = xy.shape[0]
    pts = torch.as_tensor(np.ascontiguousarray(xy, dtype=np.float64), device=DEV)
    out = torch.full((n,), float("nan"), dtype=torch.float64, device=DEV)
    ext.lidar_density(lidar.cuda_args(DEV), pts.data_ptr(), n, out.data_ptr())
    return out.cpu().numpy()


def _query_points(lidar, rng):
    """Uniform points of the domain, every knot in x and in y (the repeated end knots included), grid nodes, and
    points beyond each side and each corner."""
    tx, ty = lidar.density.get_knots()
    x0, x1, y0, y1 = lidar.xs[0], lidar.xs[-1], lidar.ys[0], lidar.ys[-1]
    uni = np.stack([rng.uniform(x0, x1, 100000), rng.uniform(y0, y1, 100000)], 1)
    kx = np.stack([tx, rng.uniform(y0, y1, tx.size)], 1)
    ky = np.stack([rng.uniform(x0, x1, ty.size), ty], 1)
    kk = np.stack(np.meshgrid(np.r_[tx[:6], tx[-6:]], np.r_[ty[:6], ty[-6:]]), -1).reshape(-1, 2)
    far = []
    for d in (1e-9, 0.3, 7.0, 1e4):
        for sx in (-1, 0, 1):
            for sy in (-1, 0, 1):
                if sx == sy == 0:
                    continue
                x = {-1: x0 - d, 1: x1 + d, 0: rng.uniform(x0, x1)}[sx]
                y = {-1: y0 - d, 1: y1 + d, 0: rng.uniform(y0, y1)}[sy]
                far.append((x, y))
    return np.concatenate([uni, kx, ky, kk, np.asarray(far)])


def _grid_nodes(lidar, rng, n=20000):
    i = np.r_[0, lidar.nx - 1, rng.integers(0, lidar.nx, n)]
    j = np.r_[lidar.ny - 1, 0, rng.integers(0, lidar.ny, n)]
    return np.stack([lidar.xs[i], lidar.ys[j]], 1), lidar.img[j, i]


def _plans(tmp):
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    write_dataset(tmp, n_paths=1, seed=1)
    noise = np.random.default_rng(3).integers(0, 256, size=(37, 53)).astype(float) / 255.0
    return {"reference": _paper_lidar(),
            "synthetic": Lidar2D(os.path.join(tmp, "floor_img.png"), 8, 0.2, 10, 1.0, 20, 3, border_width=8),
            "noise_37x53": Lidar2D(noise, 8, 0.2, 10, 1.0, 20, 3, border_width=0)}


def test_density_matches_fitpack(tmp_path):
    """``lidar_density`` within 1e-12 of ``RectBivariateSpline.ev`` (FITPACK, fp64), which clamps outside the domain
    as the kernel does; at grid nodes the interpolating spline equals the image.  Point counts 1, 255, 257 and the
    whole set (~100k) cover a partial 256-thread block on either side of one."""
    rng = np.random.default_rng(0)
    for name, lidar in _plans(str(tmp_path)).items():
        pts = _query_points(lidar, rng)
        ref = lidar.density.ev(pts[:, 0], pts[:, 1])
        got = _density_gpu(lidar, pts)
        err = np.abs(got - ref)
        assert err.max() <= 1e-12, (name, err.max(), pts[err.argmax()])
        perm = rng.permutation(pts.shape[0])
        for n in (1, 255, 257):
            sel = perm[:n]
            np.testing.assert_allclose(_density_gpu(lidar, pts[sel]), ref[sel], rtol=0, atol=1e-12, err_msg=name)
        nodes, img = _grid_nodes(lidar, rng)
        got = _density_gpu(lidar, nodes)
        np.testing.assert_allclose(got, lidar.density.ev(nodes[:, 0], nodes[:, 1]), rtol=0, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(got, img, rtol=0, atol=1e-9, err_msg=name)


def test_density_of_no_points_launches_nothing():
    lidar = _paper_lidar()
    out = torch.zeros(1, dtype=torch.float64, device=DEV)
    load_ext(required=True).lidar_density(lidar.cuda_args(DEV), 0, 0, out.data_ptr())
    torch.cuda.synchronize()
    assert out.item() == 0.0


# ---- the scans ----------------------------------------------------------------------------------------------------
def _oracle_march(lidar, pos):
    """Coarse hit index of every beam and the smallest |density - 0.5| over every coarse and fine sample, as
    ``_scan_chunk`` computes them."""
    P, Bm = pos.shape[0], lidar.num_beams
    bv = lidar._beam_vectors()
    tc = np.linspace(0.0, 1.0, lidar.collision_samps)
    coarse = pos[:, None, None, :] + tc[None, None, :, None] * bv[None, :, None, :]
    cvals = lidar.density.ev(coarse[..., 0].ravel(), coarse[..., 1].ravel()).reshape(P, Bm, -1)
    hit = np.argmax(cvals >= THR, axis=2)
    margin = np.abs(cvals - THR).min()
    pi, bi = np.nonzero(hit > 0)
    if pi.size:
        coll, last = coarse[pi, bi, hit[pi, bi]], coarse[pi, bi, hit[pi, bi] - 1]
        tf = np.linspace(0.0, 1.0, lidar.fine_samps)
        fine = last[:, None, :] + tf[None, :, None] * (coll - last)[:, None, :]
        fvals = lidar.density.ev(fine[..., 0].ravel(), fine[..., 1].ravel())
        margin = min(margin, np.abs(fvals - THR).min())
    return hit, margin


def _check_scans(lidar, pos, atol=1e-9):
    """GPU scans of ``pos`` against the NumPy twin; returns the oracle's coarse hit indices."""
    pos = np.asarray(pos, dtype=float).reshape(-1, 2)
    hit, margin = _oracle_march(lidar, pos)
    assert margin > 1e-9, f"ill-posed case: a sample lies {margin:.1e} from the threshold"
    cpu = lidar.scan_batch(pos)
    gpu = lidar.scan_batch(pos, device=DEV)
    assert gpu.shape == cpu.shape == (pos.shape[0], lidar.num_beams * lidar.beam_samps, 3)
    assert np.isfinite(gpu).all()
    err = np.abs(gpu - cpu).max(axis=(0, 1)) if gpu.size else np.zeros(3)
    assert (err <= atol).all(), f"max |gpu - cpu| in (x, y, density): {err}"
    return hit


def test_scans_match_reference_golden_scans():
    """The reference's own per-beam scans on its floor plan (tests/test_properties.py holds the NumPy path to the
    same bar)."""
    golden = np.load(os.path.join(ROOT, "tests", "golden", "reference_optimizers.npz"))
    lidar = Lidar2D(PLAN, 12, 0.2, 15, 1.0, 30, 3, border_width=30)
    traj = _trajectory(lidar, 1)[::6]
    gpu = lidar.scan_batch(traj, device=DEV)
    np.testing.assert_allclose(gpu, golden["lidar/scans"], rtol=1e-9, atol=1e-9)


def test_scans_on_the_paper_trajectory():
    """dist_online_dense_PAPER's lidar along tight_paths/1 at spline_res 30: 2430 poses x 20 beams = 48 600 threads,
    the last block partial; beams with and without a hit."""
    lidar = _paper_lidar()
    pos = _trajectory(lidar)
    assert pos.shape == (2430, 2)
    hit = _check_scans(lidar, pos)
    assert (hit == 0).any() and (hit > 1).any()


def test_scans_on_a_synthetic_plan(tmp_path):
    """A generated floor plan and trajectory with samp_df 1.3."""
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path)
    write_dataset(d, n_paths=2, seed=1)
    lidar = Lidar2D(os.path.join(d, "floor_img.png"), 20, 0.2, 25, 1.3, 50, 3, border_width=8)
    wp = np.load(os.path.join(d, "tight_paths", "1.npy"))
    traj = interpolate_waypoints(wp[:, 0], wp[:, 1], 6) * np.array([lidar.nx * 0.5, lidar.ny * 0.5])
    hit = _check_scans(lidar, traj)
    assert (hit == 0).any() and (hit > 0).any()


def _near_wall_poses(lidar, n=24):
    """Free poses of the reference plan within one coarse step of a wall: some beam hits at coarse sample 1."""
    rng = np.random.default_rng(11)
    x = rng.uniform(lidar.xs[0], lidar.xs[-1], 4000)
    y = rng.uniform(lidar.ys[0], lidar.ys[-1], 4000)
    free = lidar.density.ev(x, y) < 0.45
    pos = np.stack([x[free], y[free]], 1)
    hit, _ = _oracle_march(lidar, pos)
    return pos[(hit == 1).any(1)][:n]


def test_scans_hitting_at_the_first_coarse_sample():
    """hit == 1: the fine search starts at the pose itself."""
    lidar = _paper_lidar()
    pos = _near_wall_poses(lidar)
    assert pos.shape[0] == 24
    hit = _check_scans(lidar, pos)
    assert (hit == 1).sum() >= 24


def _box_image():
    img = np.zeros((90, 140))
    img[30:55, 60:100] = 1.0
    return img


def test_scans_leaving_the_image():
    """No border and beams as long as the image: beams that miss the box end outside the domain, where the spline is
    evaluated clamped at its end knots."""
    lidar = Lidar2D(_box_image(), 16, 1.0, 20, 1.3, 40, 5, border_width=0)
    pos = np.array([[-50.0, -30.0], [-60.0, 35.0], [10.0, -40.0], [60.0, 35.0], [-5.0, 38.0]])
    hit = _check_scans(lidar, pos)
    assert (hit == 0).any() and (hit > 0).any()
    end = pos[:, None, :] + lidar._beam_vectors()[None]
    out = (np.abs(end[..., 0]) > lidar.xs[-1]) | (np.abs(end[..., 1]) > lidar.ys[-1])
    assert out[hit == 0].all()


def test_scans_of_an_empty_image():
    """No beam collides: the samples stay evenly spaced even with samp_df != 1."""
    lidar = Lidar2D(np.zeros((50, 70)), 9, 0.4, 11, 2.0, 30, 3, border_width=0)
    pos = np.array([[0.0, 0.0], [-20.0, 10.0], [30.0, -20.0]])
    hit = _check_scans(lidar, pos)
    assert (hit == 0).all()


@pytest.mark.parametrize("samp_df", [0.5, 1.0, 1.3, 2.0])
def test_scans_at_every_sample_exponent(samp_df):
    lidar = _variant(_paper_lidar(), samp_df=samp_df)
    _check_scans(lidar, _trajectory(lidar)[::97])


@pytest.mark.parametrize("P", [1, 3, 127])
@pytest.mark.parametrize("num_beams", [1, 7, 128, 129])
def test_scans_at_any_beam_and_pose_count(num_beams, P):
    """P x num_beams threads fill a 128-thread block exactly, partly, or spill one thread into the next."""
    lidar = _variant(_paper_lidar(), num_beams=num_beams)
    pos = _trajectory(lidar)[5::19][:P]
    _check_scans(lidar, pos)


@pytest.mark.parametrize("which", ["collision_samps", "fine_samps", "beam_samps"])
@pytest.mark.parametrize("count", [1, 2])
def test_scans_with_the_fewest_samples(which, count):
    """Two samples: the coarse march tests only the pose and the beam end, the fine search only the two coarse samples
    around the hit, the output only the pose and the end point.  One sample sits at t = 0, as np.linspace(0, 1, 1)
    puts it: no collision from one coarse sample, the last empty point as the fine end point, the pose as the only
    output sample (not NaN from 0 * (1 / 0))."""
    base = _paper_lidar()
    lidar = _variant(base, **{which: count})
    pos = np.concatenate([_trajectory(lidar)[::61], _near_wall_poses(base, 6)])
    hit = _check_scans(lidar, pos)
    if which != "collision_samps":
        assert (hit > 0).any()


def test_scans_of_no_poses():
    """Zero poses: an empty result of the CPU path's shape, and no launch."""
    lidar = _paper_lidar()
    pos = np.zeros((0, 2))
    gpu = lidar.scan_batch(pos, device=DEV)
    torch.cuda.synchronize()
    assert gpu.shape == lidar.scan_batch(pos).shape == (0, lidar.num_beams * lidar.beam_samps, 3)
