// The PPO update of every node at once (rl/dist_ppo.py, rl/ppo.py): per-node normalised advantages, and the actor and
// critic losses and gradients of one primal step.
//
// Decomposition: actor and critic share no parameters, so a CTA owns one (node, network, chunk of the node's samples)
// and walks its chunk in tiles of `tm` rows: obs tile -> forward (ReLU hidden layers, linear output) -> per-row loss
// and output gradient -> backward.  Every contraction is a warp-level 16 x 16 tile on the tensor cores: fp64 DMMA
// m16n8k4, fp32 3xTF32 m16n8k8 (common.cuh).  Widths are padded to multiples of 16 with zeros (obs_dim 12 -> 16, the
// 5- and 1-wide outputs -> 16); weights are read in place through L1, guarded, so arena rows work directly.
//
// Gradients: dW_l += dZ_l^T H_l accumulates across the CTA's tiles in double in shared memory (each element owned by
// one warp lane per tile), db_l by one thread per output; each CTA writes one partial slot and ppo_reduce_kernel sums
// the chunks' slots in a fixed order straight into the per-layer gradient tensors, parameter ranges only.
// Nothing is atomic in any sum, so two launches are bitwise equal.
//
// The per-row loss terms are evaluated in double (exp and division are correctly rounded whatever --use_fast_math
// does to fp32), with autograd's clip semantics: torch.min splits a tie evenly and clamp passes the gradient on the
// closed interval, so d actor_loss / d r = -A / R when r is in [1 - clip, 1 + clip] or r A < clamp(r) A, else 0.
#include <map>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "ppo_update.h"

namespace nndt {
namespace ppo {

namespace {

constexpr int NT = 256, NWARP = NT / kWarp, PADE = 4;   // threads per CTA, row padding of the activation tiles

__host__ __device__ inline int pad16(int x) { return (x + 15) & ~15; }

// Shared memory of one network's CTA: gradient accumulators G_l [P_{l+1}][P_l] + db_l [P_{l+1}] in double (backward
// only; offsets goff in doubles), then from byte hbase the activation tiles H_l [tm][P_l + PADE] in T for l = 0..nl
// (H_nl = output; offsets hoff in elements of T), then tm doubles of row losses.
struct Layout {
  int P[kMaxLayers + 1], ld[kMaxLayers + 1];
  size_t goff[kMaxLayers], hoff[kMaxLayers + 1], gsize, hbase, rowloss, bytes;
};
__host__ __device__ inline Layout layout(const int* dims, int nl, int tm, bool bwd, size_t es) {
  Layout L;
  size_t o = 0;
  for (int l = 0; l <= nl; ++l) {
    L.P[l] = pad16(dims[l]);
    L.ld[l] = L.P[l] + PADE;
  }
  for (int l = 0; l < nl; ++l) {
    L.goff[l] = o;
    o += (size_t)L.P[l + 1] * L.P[l] + L.P[l + 1];
  }
  L.gsize = o;
  L.hbase = bwd ? L.gsize * sizeof(double) : 0;
  o = 0;
  for (int l = 0; l <= nl; ++l) {
    L.hoff[l] = o;
    o += (size_t)tm * L.ld[l];
  }
  L.rowloss = (L.hbase + o * es + 7) & ~(size_t)7;
  L.bytes = L.rowloss + (size_t)tm * sizeof(double);
  return L;
}

NNDT_DEVINL float add_rn(float x, float y) { return __fadd_rn(x, y); }
NNDT_DEVINL double add_rn(double x, double y) { return __dadd_rn(x, y); }
NNDT_DEVINL float sub_rn(float x, float y) { return __fsub_rn(x, y); }
NNDT_DEVINL double sub_rn(double x, double y) { return __dsub_rn(x, y); }
NNDT_DEVINL float mul_rn(float x, float y) { return __fmul_rn(x, y); }
NNDT_DEVINL double mul_rn(double x, double y) { return __dmul_rn(x, y); }
template <typename T> NNDT_DEVINL T div_rn(T x, T y);
template <> NNDT_DEVINL float div_rn(float x, float y) { return __fdiv_rn(x, y); }
template <> NNDT_DEVINL double div_rn(double x, double y) { return __ddiv_rn(x, y); }

template <typename T>
NNDT_DEVINL void zero_acc(T (&c)[2][4]) {
#pragma unroll
  for (int j = 0; j < 2; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = (T)0;
}

// One CTA = (chunk, network net0 + blockIdx.y, node blockIdx.z).  BWD = false is the advantage pass: critic forward
// only, writing A = rtgs - V, or V itself for gae_kernel when GAE is requested.
template <typename T, bool BWD>
__global__ void __launch_bounds__(NT, 1) ppo_grad_kernel(const Args a, const int tm, const int chunks, const int net0,
                                                      const size_t gmax, double* gpart, double* lpart) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // the layout, shape and pointers are indexed by layer at run time: keep them in shared memory, not on the stack
  __shared__ Layout L;
  __shared__ Net nw;
  __shared__ int dims[kMaxLayers + 1];
  const int chunk = blockIdx.x, net = net0 + blockIdx.y, node = blockIdx.z;
  const int nl = a.nl[net];
  if (threadIdx.x == 0) {
    L = layout(a.dims[net], nl, tm, BWD, sizeof(T));
    nw = a.net[node][net];
    for (int l = 0; l <= nl; ++l) dims[l] = a.dims[net][l];
  }
  __syncthreads();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, mt = tm / 16;
  const int R = a.R, din0 = dims[0];
  const int per = ((R + chunks - 1) / chunks + tm - 1) / tm * tm;
  const int r0 = chunk * per, r1 = min(R, r0 + per);
  double* G = reinterpret_cast<double*>(smem_raw);
  T* sm = reinterpret_cast<T*>(smem_raw + L.hbase);
  double* rowloss = reinterpret_cast<double*>(smem_raw + L.rowloss);
  if (BWD)
    for (size_t q = tid; q < L.gsize; q += NT) G[q] = 0.0;
  for (int q = tid; q < tm; q += NT) rowloss[q] = 0.0;
  const T* obs = reinterpret_cast<const T*>(a.obs) + (size_t)node * R * din0;
  const size_t nrow0 = (size_t)node * R;
  __syncthreads();

  for (int row0 = r0; row0 < r1; row0 += tm) {
    const int rows = min(tm, r1 - row0);
    {
      T* H0 = sm + L.hoff[0];
      for (int q = tid; q < tm * L.P[0]; q += NT) {
        const int m = q / L.P[0], k = q - m * L.P[0];
        H0[m * L.ld[0] + k] = (m < rows && k < din0) ? obs[(size_t)(row0 + m) * din0 + k] : (T)0;
      }
    }
    __syncthreads();

    // ---- forward: H_{l+1} = act(H_l W_l^T + b_l)
    for (int l = 0; l < nl; ++l) {
      const int din = dims[l], dout = dims[l + 1], ldx = L.ld[l], ldy = L.ld[l + 1];
      const T* W = reinterpret_cast<const T*>(nw.W[l]);
      const T* B = reinterpret_cast<const T*>(nw.b[l]);
      const T* X = sm + L.hoff[l];
      T* Y = sm + L.hoff[l + 1];
      const bool relu = l + 1 < nl;
      const auto w_kn = [W, din, dout](int k, int n) { return (k < din && n < dout) ? __ldg(W + n * din + k) : (T)0; };
      for (int w = warp; w < mt * (L.P[l + 1] / 16); w += NWARP) {
        const int m0 = (w % mt) * 16, n0 = (w / mt) * 16;
        T c[2][4];
        zero_acc(c);
        gemm<2>(c, m0, n0, L.P[l], lane, at(X, ldx), w_kn);
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = frow(m0, lane, i), col = fcol(n0 + 8 * j, lane, i);
            const T z = c[j][i] + (col < dout ? __ldg(B + col) : (T)0);
            Y[row * ldy + col] = relu && z < (T)0 ? (T)0 : z;   // a NaN passes the ReLU, as in torch
          }
      }
      __syncthreads();
    }

    // ---- per-row loss and output gradient dZ (in place of the output tile)
    if (tid < tm) {
      const int m = tid;
      const size_t r = nrow0 + row0 + m;
      T* O = sm + L.hoff[nl] + m * L.ld[nl];
      double loss = 0.0;
      if (m < rows) {
        if (net == kActor) {
          const T* act = reinterpret_cast<const T*>(a.acts) + r * kActDim;
          double d[kActDim], S = 0.0;
          bool finite = true;
#pragma unroll
          for (int k = 0; k < kActDim; ++k) {
            const double mean = (double)O[k];
            finite = finite && isfinite(mean);
            d[k] = (double)act[k] - mean;
            S += d[k] * d[k];
          }
          if (!finite) *a.nonfinite = 1;
          const double lp = -0.5 * S / a.cov_var - a.lp_const;
          const double ratio = exp(lp - (double)reinterpret_cast<const T*>(a.old_lp)[r]);
          const double A = (double)reinterpret_cast<const T*>(a.adv)[r];
          const double lo = 1.0 - a.clip, hi = 1.0 + a.clip;
          const double s1 = ratio * A, s2 = fmin(fmax(ratio, lo), hi) * A;
          loss = -fmin(s1, s2);
          if (BWD) {
            const double gr = (ratio >= lo && ratio <= hi) || s1 < s2 ? -A * ratio / ((double)R * a.cov_var) : 0.0;
#pragma unroll
            for (int k = 0; k < kActDim; ++k) O[k] = (T)(gr * d[k]);
          }
        } else {
          const T rtg = reinterpret_cast<const T*>(a.rtgs)[r];
          const double e = (double)O[0] - (double)rtg;
          loss = e * e;
          if (BWD) O[0] = (T)(2.0 * e / (double)R);
          else reinterpret_cast<T*>(a.adv)[r] = a.gae ? O[0] : rtg - O[0];
        }
      } else if (BWD) {
        for (int k = 0; k < L.P[nl]; ++k) O[k] = (T)0;   // rows past the chunk contribute nothing
      }
      rowloss[m] += loss;
    }
    if (!BWD) {
      __syncthreads();
      continue;
    }
    __syncthreads();

    // ---- backward: dW_l += dZ_l^T H_l, db_l += sum_m dZ_l, dZ_{l-1} = (dZ_l W_l) * (H_l > 0) in place of H_l.  A tile's
    // contribution is formed in T on the tensor cores and added to the double accumulators, so the sum over the
    // thousands of tiles of a chunk does not lose fp32 digits.
    for (int l = nl - 1; l >= 0; --l) {
      const int din = dims[l], dout = dims[l + 1], Pi = L.P[l], Po = L.P[l + 1], ldx = L.ld[l], ldd = L.ld[l + 1];
      T* X = sm + L.hoff[l];
      const T* D = sm + L.hoff[l + 1];
      double* Gl = G + L.goff[l];
      for (int w = warp; w < (Po / 16) * (Pi / 16); w += NWARP) {
        const int m0 = (w % (Po / 16)) * 16, n0 = (w / (Po / 16)) * 16;
        T c[2][4];
        zero_acc(c);
        gemm<2>(c, m0, n0, tm, lane, at_t(D, ldd), at(static_cast<const T*>(X), ldx));
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int i = 0; i < 4; ++i) Gl[frow(m0, lane, i) * Pi + fcol(n0 + 8 * j, lane, i)] += (double)c[j][i];
      }
      for (int n = tid; n < dout; n += NT) {
        double s = 0.0;
        for (int m = 0; m < tm; ++m) s += (double)D[m * ldd + n];
        Gl[(size_t)Po * Pi + n] += s;
      }
      if (l > 0) {
        __syncthreads();   // dW has read H_l
        const T* W = reinterpret_cast<const T*>(nw.W[l]);
        const auto w_nk = [W, din, dout](int n, int k) { return (n < dout && k < din) ? __ldg(W + n * din + k) : (T)0; };
        for (int w = warp; w < mt * (Pi / 16); w += NWARP) {
          const int m0 = (w % mt) * 16, n0 = (w / mt) * 16;
          T c[2][4];
          zero_acc(c);
          gemm<2>(c, m0, n0, Po, lane, at(D, ldd), w_nk);
#pragma unroll
          for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              T* h = X + frow(m0, lane, i) * ldx + fcol(n0 + 8 * j, lane, i);
              *h = *h > (T)0 ? c[j][i] : (T)0;
            }
        }
      }
      __syncthreads();
    }
  }

  if (!BWD) return;
  const size_t slot = ((size_t)node * 2 + net) * chunks + chunk;
  for (size_t q = tid; q < L.gsize; q += NT) gpart[slot * gmax + q] = G[q];
  if (tid == 0) {
    double s = 0.0;
    for (int m = 0; m < tm; ++m) s += rowloss[m];
    lpart[slot] = s;
  }
}

// Sum of the chunks' partial slots, chunk by chunk, into the parameter ranges of the gradient tensors; losses / R.
template <typename T>
__global__ void __launch_bounds__(NT) ppo_reduce_kernel(const Args a, const int chunks, const size_t gmax,
                                                        const double* gpart, const double* lpart) {
  __shared__ Layout L;
  __shared__ Net nw;
  __shared__ int dims[kMaxLayers + 1];
  const int net = blockIdx.y, node = blockIdx.z, nl = a.nl[net];
  if (threadIdx.x == 0) {
    L = layout(a.dims[net], nl, 16, true, sizeof(T));
    nw = a.net[node][net];
    for (int l = 0; l <= nl; ++l) dims[l] = a.dims[net][l];
  }
  __syncthreads();
  const size_t base = ((size_t)node * 2 + net) * chunks;
  for (size_t q = (size_t)blockIdx.x * NT + threadIdx.x; q < L.gsize; q += (size_t)gridDim.x * NT) {
    int l = 0;
    while (l + 1 < nl && q >= L.goff[l + 1]) ++l;
    const size_t o = q - L.goff[l];
    const int Pi = L.P[l], din = dims[l], dout = dims[l + 1];
    T* dst;
    if (o < (size_t)L.P[l + 1] * Pi) {
      const int n = (int)(o / Pi), k = (int)(o - (size_t)n * Pi);
      if (n >= dout || k >= din) continue;
      dst = reinterpret_cast<T*>(nw.gW[l]) + n * din + k;
    } else {
      const int n = (int)(o - (size_t)L.P[l + 1] * Pi);
      if (n >= dout) continue;
      dst = reinterpret_cast<T*>(nw.gb[l]) + n;
    }
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += gpart[(base + c) * gmax + q];
    *dst = (T)s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += lpart[base + c];
    reinterpret_cast<T*>(a.losses)[node * 2 + net] = (T)(s / (double)a.R);
  }
}

NNDT_DEVINL double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = NT / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// One CTA per node: adv <- (A - mean) / (std + 1e-10) with the mean and unbiased std of the node's A taken in double in
// a fixed order (R = 1 gives NaN, as torch's std does).  The normalisation itself is in T, as in the torch expression.
template <typename T>
__global__ void __launch_bounds__(NT) adv_norm_kernel(T* adv, const int R) {
  __shared__ double red[NT];
  T* A = adv + (size_t)blockIdx.x * R;
  double s = 0.0;
  for (int r = threadIdx.x; r < R; r += NT) s += (double)A[r];
  const double mean = block_sum(s, red) / (double)R;
  double v = 0.0;
  for (int r = threadIdx.x; r < R; r += NT) {
    const double d = (double)A[r] - mean;
    v += d * d;
  }
  const double var = block_sum(v, red) / (double)(R - 1);
  const T mt = (T)mean, den = (T)sqrt(var) + (T)1e-10;
  for (int r = threadIdx.x; r < R; r += NT) A[r] = div_rn<T>(A[r] - mt, den);
}

// GAE(lambda), one thread per (node, episode block, world): a backward scan over the block's T cycles,
//   delta_c = r_c + gamma V_{c+1} - V_c,  A_c = delta_c + (gamma lam) A_{c+1},  G_c = A_c + V_c,  V_T = A_T = 0,
// with V read from adv (the critic pass's output) and overwritten by A, and copied to `values` when given.  Every product and sum is rounded on its own
// (no FMA contraction), in the order written, as the rewards-to-go scan of the rollout kernel is: the torch path's
// elementwise ops give the same bits.  gl = gamma * lam is rounded in double, then to T, as torch rounds a Python
// scalar.
template <typename T>
__global__ void __launch_bounds__(NT) gae_kernel(const T* rews, T* adv, T* returns, T* values, const int R,
                                                 const int steps, const int E, const double gamma, const double gl,
                                                 const int lanes) {
  const int q = blockIdx.x * NT + threadIdx.x;   // (node, block, world) of the N * (R / (T * E)) * E scans
  if (q >= lanes) return;
  const int per = R / steps;                     // scans per node: (R / (T * E)) * E
  const int node = q / per, k = q - node * per, blk = k / E, e = k - blk * E;
  const size_t base = (size_t)node * R + (size_t)blk * steps * E + e;
  const T g = (T)gamma, l = (T)gl;
  T A = (T)0, vn = (T)0;
  for (int c = steps - 1; c >= 0; --c) {
    const size_t r = base + (size_t)c * E;
    const T v = adv[r];
    const T delta = sub_rn(add_rn(rews[r], mul_rn(g, vn)), v);
    A = add_rn(delta, mul_rn(l, A));
    adv[r] = A;
    returns[r] = add_rn(A, v);
    if (values) values[r] = v;
    vn = v;
  }
}

template <typename T>
size_t gmax_of(const Args& a, int tm) {
  size_t gmax = 0;
  for (int n = 0; n < 2; ++n) {
    const size_t g = layout(a.dims[n], a.nl[n], tm, true, sizeof(T)).gsize;
    gmax = g > gmax ? g : gmax;
  }
  return gmax;
}

// The launch plan of one (device, dtype, pass, shapes, N, R); the device queries, the shared-memory opt-in and the
// occupancy query run once per key, not once per primal step.
template <typename T, bool BWD>
Plan setup(const Args& a, int dev) {
  Plan p{};
  const int nets = BWD ? 2 : 1, net0 = BWD ? kActor : kCritic;
  int nsm = 132, optin = 227 * 1024;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  auto bytes = [&](int tm) {
    size_t b = 0;
    for (int n = net0; n < net0 + nets; ++n) {
      const size_t x = layout(a.dims[n], a.nl[n], tm, BWD, sizeof(T)).bytes;
      b = x > b ? x : b;
    }
    return b;
  };
  auto kern = ppo_grad_kernel<T, BWD>;
  cudaFuncAttributes fa{};
  p.err = cudaFuncGetAttributes(&fa, kern);
  if (p.err != cudaSuccess) return p;
  const size_t dyn = (size_t)optin - fa.sharedSizeBytes;   // the opt-in covers static + dynamic shared memory
  p.tm = bytes(32) <= dyn ? 32 : 16;
  p.smem = bytes(p.tm);
  p.err = cudaErrorInvalidValue;
  if (p.smem > dyn) return p;
  // the opt-in is a per-kernel maximum: set it to the device's limit, so every cached plan stays launchable
  p.err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
  if (p.err != cudaSuccess) return p;
  int occ = 1;
  p.err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, NT, p.smem);
  if (p.err != cudaSuccess) return p;
  const int want = (nsm * (occ > 0 ? occ : 1)) / (a.N * nets), most = (a.R + p.tm - 1) / p.tm;
  p.chunks = want < 1 ? 1 : (want > most ? most : want);
  if (BWD) {
    for (int n = 0; n < 2; ++n) {
      const size_t g = layout(a.dims[n], a.nl[n], p.tm, true, sizeof(T)).gsize;
      p.gmax = g > p.gmax ? g : p.gmax;
    }
    const size_t slots = (size_t)a.N * 2 * p.chunks;
    p.work_bytes = (slots * p.gmax + slots) * sizeof(double);
  }
  return p;
}

template <typename T>
cudaError_t grads_t(const Args& a, const Plan& p, void* work, cudaStream_t st) {
  const size_t slots = (size_t)a.N * 2 * p.chunks;
  double* gpart = reinterpret_cast<double*>(work);
  double* lpart = gpart + slots * p.gmax;
  ppo_grad_kernel<T, true><<<dim3(p.chunks, 2, a.N), NT, p.smem, st>>>(a, p.tm, p.chunks, kActor, p.gmax, gpart, lpart);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int bx = (int)((p.gmax + NT - 1) / NT);
  ppo_reduce_kernel<T><<<dim3(bx, 2, a.N), NT, 0, st>>>(a, p.chunks, p.gmax, gpart, lpart);
  return cudaGetLastError();
}

template <typename T>
cudaError_t advantages_t(const Args& a, const Plan& p, cudaStream_t st) {
  ppo_grad_kernel<T, false><<<dim3(p.chunks, 1, a.N), NT, p.smem, st>>>(a, p.tm, p.chunks, kCritic, 0, nullptr, nullptr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (a.gae) {
    const int lanes = a.N * (a.R / a.T);
    gae_kernel<T><<<(lanes + NT - 1) / NT, NT, 0, st>>>(reinterpret_cast<const T*>(a.rews), reinterpret_cast<T*>(a.adv),
                                                        reinterpret_cast<T*>(a.returns),
                                                        reinterpret_cast<T*>(a.values), a.R, a.T, a.E, a.gamma,
                                                        a.gamma * a.lam, lanes);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  adv_norm_kernel<T><<<a.N, NT, 0, st>>>(reinterpret_cast<T*>(a.adv), a.R);
  return cudaGetLastError();
}

}  // namespace

const char* check(const Args& a, bool with_actor) {
  if (a.N < 1 || a.N > kMaxNodes) return "needs 1..8 nodes";
  if (a.R < 1) return "needs at least one sample per node";
  for (int n = with_actor ? kActor : kCritic; n < 2; ++n) {
    if (a.nl[n] < 1 || a.nl[n] > kMaxLayers) return "needs networks with 1..5 linear layers";
    for (int l = 0; l <= a.nl[n]; ++l)
      if (a.dims[n][l] < 1 || a.dims[n][l] > kMaxWidth) return "network widths must be 1..64";
    for (int i = 0; i < a.N; ++i)
      for (int l = 0; l < a.nl[n]; ++l)
        if (!a.net[i][n].W[l] || !a.net[i][n].b[l]) return "missing network parameter";
  }
  if (a.dims[kCritic][a.nl[kCritic]] != 1) return "critic output width != 1";
  if (!a.obs || !a.rtgs || !a.adv) return "missing buffer";
  if (a.gae) {
    if (!a.rews || !a.returns) return "missing buffer";
    if (a.T < 1 || a.E < 1 || a.R % a.T || (a.R / a.T) % a.E) return "GAE needs T * E to divide R";
    if (!(a.gamma >= 0.0 && a.gamma <= 1.0) || !(a.lam >= 0.0 && a.lam <= 1.0)) return "GAE needs gamma and lam in [0, 1]";
  }
  if (!with_actor) return nullptr;
  if (a.dims[kActor][0] != a.dims[kCritic][0]) return "actor and critic input widths differ";
  if (a.dims[kActor][a.nl[kActor]] != kActDim) return "actor output width != 5";
  if (!a.acts || !a.old_lp || !a.losses || !a.nonfinite) return "missing buffer";
  for (int i = 0; i < a.N; ++i)
    for (int n = 0; n < 2; ++n)
      for (int l = 0; l < a.nl[n]; ++l)
        if (!a.net[i][n].gW[l] || !a.net[i][n].gb[l]) return "missing gradient tensor";
  if (!(a.cov_var > 0.0) || !(a.clip >= 0.0)) return "needs cov_var > 0 and clip >= 0";
  return nullptr;
}

Plan plan(const Args& a, bool backward) {
  static std::mutex mu;
  static std::map<std::vector<int>, Plan> cache;
  int dev = 0;
  cudaGetDevice(&dev);
  std::vector<int> key{dev, a.dtype64, (int)backward, a.N, a.R};
  for (int n = backward ? kActor : kCritic; n < 2; ++n)
    for (int l = 0; l <= a.nl[n]; ++l) key.push_back(a.dims[n][l]), key.push_back(n);
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  const Plan p = a.dtype64 ? (backward ? setup<double, true>(a, dev) : setup<double, false>(a, dev))
                           : (backward ? setup<float, true>(a, dev) : setup<float, false>(a, dev));
  if (p.err == cudaSuccess) cache.emplace(key, p);
  return p;
}

cudaError_t grads(const Args& a, const Plan& p, void* work, cudaStream_t st) {
  if (check(a, true)) return cudaErrorInvalidValue;
  if (p.err != cudaSuccess) return p.err;
  return a.dtype64 ? grads_t<double>(a, p, work, st) : grads_t<float>(a, p, work, st);
}

cudaError_t advantages(const Args& a, cudaStream_t st) {
  if (check(a, false)) return cudaErrorInvalidValue;
  const Plan p = plan(a, false);
  if (p.err != cudaSuccess) return p.err;
  return a.dtype64 ? advantages_t<double>(a, p, st) : advantages_t<float>(a, p, st);
}

}  // namespace ppo
}  // namespace nndt
