// Batched 2-D lidar scans on the GPU: one thread per (pose, beam) marches the beam through the
// bicubic B-spline density field (the same tensor-product spline scipy's RectBivariateSpline fits;
// knots and coefficients are uploaded from it), refines the collision point and emits the beam's
// samples.  Reference: floorplans/lidar/lidar.py:61-136, which runs this per pose and per beam in
// Python (minutes for a robot's ~2 400 scans).  fp64 throughout: results match the CPU path to 1e-10.
#include "common.cuh"
#include "lidar.h"

namespace nndt {
namespace lidar {

struct Spline {
  const double* tx; const double* ty; const double* c;
  int ntx, nty;          // number of knots; coefficient grid is (ntx-4) x (nty-4)
};

__device__ __forceinline__ int find_span(const double* t, int nt, double x) {
  // largest i in [3, nt-5] with t[i] <= x   (x already clamped to [t[3], t[nt-4]])
  int lo = 3, hi = nt - 5;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ void basis(const double* t, int i, double x, double (&N)[4]) {
  double left[4], right[4];
  N[0] = 1.0;
#pragma unroll
  for (int j = 1; j <= 3; ++j) {
    left[j] = x - t[i + 1 - j];
    right[j] = t[i + j] - x;
    double saved = 0.0;
#pragma unroll
    for (int r = 0; r < j; ++r) {
      const double temp = N[r] / (right[r + 1] + left[j - r]);
      N[r] = saved + right[r + 1] * temp;
      saved = left[j - r] * temp;
    }
    N[j] = saved;
  }
}

// spacing of n samples over [0, 1], as np.linspace(0, 1, n): a single sample sits at t = 0
__device__ __forceinline__ double unit_step(int n) { return n > 1 ? 1.0 / (double)(n - 1) : 0.0; }

__device__ __forceinline__ double density(const Spline& s, double x, double y) {
  x = fmin(fmax(x, s.tx[3]), s.tx[s.ntx - 4]);
  y = fmin(fmax(y, s.ty[3]), s.ty[s.nty - 4]);
  const int ix = find_span(s.tx, s.ntx, x), iy = find_span(s.ty, s.nty, y);
  double Nx[4], Ny[4];
  basis(s.tx, ix, x, Nx);
  basis(s.ty, iy, y, Ny);
  const int ncy = s.nty - 4;
  double v = 0.0;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const double* row = s.c + (size_t)(ix - 3 + a) * ncy + (iy - 3);
    v += Nx[a] * (Ny[0] * row[0] + Ny[1] * row[1] + Ny[2] * row[2] + Ny[3] * row[3]);
  }
  return v;
}

__global__ void __launch_bounds__(128) scan_kernel(const Args a) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.n_poses * a.num_beams) return;
  const int p = idx / a.num_beams, b = idx - p * a.num_beams;
  const Spline s{a.tx, a.ty, a.coef, a.ntx, a.nty};
  const double px = a.poses[2 * p], py = a.poses[2 * p + 1];
  const double ang = -M_PI + (double)b * (2.0 * M_PI / (double)a.num_beams);
  const double bx = a.beam_len * cos(ang), by = a.beam_len * sin(ang);
  const double thr = 0.5;
  // coarse march: first sample at or above the threshold (index 0 == the pose itself == "no hit")
  const double cstep = unit_step(a.collision_samps);
  int hit = 0;
  for (int i = 0; i < a.collision_samps; ++i) {
    const double t = (double)i * cstep;
    if (density(s, px + t * bx, py + t * by) >= thr) { hit = i; break; }
  }
  double ex = px + bx, ey = py + by;     // end point of the sampled segment
  const bool collided = hit > 0;
  if (collided) {
    const double t1 = (double)hit * cstep, t0 = (double)(hit - 1) * cstep;
    const double cx = px + t1 * bx, cy = py + t1 * by, lx = px + t0 * bx, ly = py + t0 * by;
    const double fstep = unit_step(a.fine_samps);
    int fh = 0;
    for (int i = 0; i < a.fine_samps; ++i) {
      const double t = (double)i * fstep;
      if (density(s, lx + t * (cx - lx), ly + t * (cy - ly)) >= thr) { fh = i; break; }
    }
    const double tf = (double)fh * fstep;
    ex = lx + tf * (cx - lx); ey = ly + tf * (cy - ly);
  }
  const double sstep = unit_step(a.beam_samps);
  double* out = a.out + ((size_t)p * a.num_beams + b) * a.beam_samps * 3;
  for (int i = 0; i < a.beam_samps; ++i) {
    double t = (double)i * sstep;
    if (collided) t = pow(t, a.samp_df);
    const double x = px + t * (ex - px), y = py + t * (ey - py);
    out[3 * i] = x; out[3 * i + 1] = y; out[3 * i + 2] = density(s, x, y);
  }
}

__global__ void density_kernel(const Args a, const double* xy, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = density(Spline{a.tx, a.ty, a.coef, a.ntx, a.nty}, xy[2 * i], xy[2 * i + 1]);
}

cudaError_t launch_scan(const Args& a, cudaStream_t st) {
  const int n = a.n_poses * a.num_beams;
  if (n <= 0) return cudaSuccess;        // no poses: nothing to scan (an empty grid is not a valid launch)
  scan_kernel<<<(n + 127) / 128, 128, 0, st>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_density(const Args& a, const double* xy, int n, double* out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  density_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, xy, n, out);
  return cudaGetLastError();
}

}  // namespace lidar
}  // namespace nndt
