// Generic conv-net forward/backward (and evaluation) on CUDA cores, fp32 or fp64, for every architecture the model
// class accepts — MNISTConvNet(num_filters <= 8, kernel_size in {3, 5}, linear_width <= 128)
// (reference: models/mnist_conv_nn.py:10-25 takes any (num_filters, kernel_size, linear_width); the whole reference runs
// in float64, experiments/dist_mnist_ex.py:19).  Two jobs:
//   * the float64 arm of the framework (same-precision comparison against the reference; fp64
//     forward/backward is DFMA work on the CUDA cores);
//   * every conv shape other than the paper's (3, 5, 64), which has the specialised kernels of mnist.cu / mnist_tc.cu.
// Same launch contract as mnist.cu: grid = (S batch slices, L nodes), in-kernel stateless sampler (or the `direct`
// staging sets of the host-fed pipeline), one partial gradient row and one loss partial per CTA, draw counters owned
// by the kernel, PDL.  fc1 weights are not staged: a CTA streams W1 from L2 three times (fc1, da1, and the dW1
// write-out), which is the right trade for a kernel whose job is coverage, not the headline.
#include "mnist_device.cuh"

namespace nndt {
namespace mnist {

namespace {

constexpr int GNT = 256;

struct Dims { int F, KS, LW, CO, PO, NP, K1; double mean, inv_std; };

__host__ __device__ inline Dims make_dims(const GenericShape& g) {
  Dims d;
  d.F = g.F; d.KS = g.KS; d.LW = g.LW;
  d.CO = HW - g.KS + 1; d.PO = d.CO / 2; d.NP = d.PO * d.PO; d.K1 = d.F * d.NP;
  d.mean = g.mean; d.inv_std = g.inv_std;
  return d;
}

template <typename T, int SPB>
struct Carve {
  T *img, *a1, *da1, *h, *dh, *z, *dz, *wc, *w2, *b1, *b2, *red, *part;
  unsigned char* arg;
  int *sidx, *label;
  float* valid;
  __host__ __device__ static size_t bytes(const Dims& d) {
    size_t n = (size_t)SPB * HW * HW + 2 * (size_t)SPB * d.K1 + 2 * (size_t)SPB * d.LW + 2 * SPB * 16 +
               (d.F * d.KS * d.KS + d.F + 4) + NCLS * d.LW + d.LW + 16 + SPB + 8 + 2 * GNT;
    return n * sizeof(T) + (size_t)SPB * d.K1 + 64 + 3 * SPB * 4 + 64;
  }
  __device__ explicit Carve(unsigned char* base, const Dims& d) {
    T* p = reinterpret_cast<T*>(base);
    img = p; p += SPB * HW * HW;
    a1 = p; p += SPB * d.K1;
    da1 = p; p += SPB * d.K1;
    h = p; p += SPB * d.LW;
    dh = p; p += SPB * d.LW;
    z = p; p += SPB * 16;
    dz = p; p += SPB * 16;
    wc = p; p += (d.F * d.KS * d.KS + d.F + 4) & ~1;
    w2 = p; p += NCLS * d.LW;
    b1 = p; p += d.LW;
    b2 = p; p += 16;
    red = p; p += (SPB + 1) & ~1;
    part = p; p += 2 * GNT;
    int* q = reinterpret_cast<int*>(p);
    sidx = q; q += SPB;
    label = q; q += SPB;
    valid = reinterpret_cast<float*>(q); q += SPB;
    arg = reinterpret_cast<unsigned char*>(q);
  }
};

template <typename T> NNDT_DEVINL T wsum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <typename T> NNDT_DEVINL T ldg(const T* p) { return __ldg(p); }
NNDT_DEVINL float gexp(float x) { return __expf(x); }
NNDT_DEVINL double gexp(double x) { return exp(x); }
NNDT_DEVINL float glog(float x) { return __logf(x); }
NNDT_DEVINL double glog(double x) { return log(x); }

// forward (+ loss, + backward when TRAIN) of the SPB samples whose indices are already in sm.sidx / sm.valid / sm.label
template <typename T, int KS, int SPB, bool TRAIN>
NNDT_DEVINL void generic_chunk(Carve<T, SPB>& sm, const Args& a, const Dims& d, const T* th, int l, int slice, int S,
                               T inv_bs, int tid) {
  constexpr int NW = GNT / 32;
  const int warp = tid >> 5, lane = tid & 31;
  // ---- pixels ---------------------------------------------------------------------------------
  for (int o = tid; o < SPB * 196; o += GNT) {
    const int s = o / 196, q = o - s * 196;
    T v0 = 0, v1 = 0, v2 = 0, v3 = 0;
    if (sm.valid[s] != 0.f) {
      const size_t base = (size_t)sm.sidx[s] * 784 + 4 * q;
      if (a.x_is_u8) {
        const uint32_t p = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const unsigned char*>(a.x) + base);
        const T mean = (T)d.mean, is = (T)d.inv_std, sc = (T)1 / (T)255;
        v0 = ((T)(p & 0xff) * sc - mean) * is;
        v1 = ((T)((p >> 8) & 0xff) * sc - mean) * is;
        v2 = ((T)((p >> 16) & 0xff) * sc - mean) * is;
        v3 = ((T)(p >> 24) * sc - mean) * is;
      } else {
        const float4 f = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.x) + base);
        v0 = (T)f.x; v1 = (T)f.y; v2 = (T)f.z; v3 = (T)f.w;
      }
    }
    T* dst = sm.img + s * 784 + 4 * q;
    dst[0] = v0; dst[1] = v1; dst[2] = v2; dst[3] = v3;
  }
  __syncthreads();
  // ---- conv + ReLU + maxpool --------------------------------------------------------------------
  for (int it = tid; it < SPB * d.K1; it += GNT) {
    const int s = it / d.K1, r = it - s * d.K1;
    const int c = r / d.NP, p = r - c * d.NP;
    const int py = p / d.PO, px = p - py * d.PO;
    const T* x = sm.img + s * 784 + (2 * py) * HW + 2 * px;
    const T* w = sm.wc + c * KS * KS;
    T a00 = 0, a01 = 0, a10 = 0, a11 = 0;
    T prev[KS + 1];
#pragma unroll
    for (int j = 0; j <= KS; ++j) prev[j] = x[j];
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
      T cur[KS + 1];
#pragma unroll
      for (int j = 0; j <= KS; ++j) cur[j] = x[(ky + 1) * HW + j];
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        const T wv = w[ky * KS + kx];
        a00 += wv * prev[kx]; a01 += wv * prev[kx + 1];
        a10 += wv * cur[kx];  a11 += wv * cur[kx + 1];
      }
#pragma unroll
      for (int j = 0; j <= KS; ++j) prev[j] = cur[j];
    }
    T m = a00; int ai = 0;                       // first maximum wins, like ATen's max_pool2d
    if (a01 > m) { m = a01; ai = 1; }
    if (a10 > m) { m = a10; ai = 2; }
    if (a11 > m) { m = a11; ai = 3; }
    m += sm.wc[d.F * KS * KS + c];
    sm.a1[it] = m > (T)0 ? m : (T)0;
    sm.arg[it] = (unsigned char)ai;
  }
  __syncthreads();
  // ---- fc1 + ReLU: one warp per output row, coalesced stream of W1 ----------------------------------
  const T* w1 = th + a.off_w1;
  for (int j = warp; j < d.LW; j += NW) {
    T acc[SPB];
#pragma unroll
    for (int s = 0; s < SPB; ++s) acc[s] = 0;
    const T* wr = w1 + (size_t)j * d.K1;
    for (int k0 = lane; k0 < d.K1; k0 += 128) {
      T wv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) wv[u] = (k0 + 32 * u < d.K1) ? ldg(wr + k0 + 32 * u) : (T)0;
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (k0 + 32 * u < d.K1) {
#pragma unroll
          for (int s = 0; s < SPB; ++s) acc[s] += wv[u] * sm.a1[s * d.K1 + k0 + 32 * u];
        }
    }
#pragma unroll
    for (int s = 0; s < SPB; ++s) acc[s] = wsum(acc[s]);
    if (lane == 0) {
      const T b = sm.b1[j];
#pragma unroll
      for (int s = 0; s < SPB; ++s) { const T v = acc[s] + b; sm.h[s * d.LW + j] = v > (T)0 ? v : (T)0; }
    }
  }
  __syncthreads();
  // ---- fc2 -------------------------------------------------------------------------------------------
  for (int o = warp; o < SPB * NCLS; o += NW) {
    const int s = o / NCLS, c = o - s * NCLS;
    T v = 0;
    for (int j = lane; j < d.LW; j += 32) v += sm.h[s * d.LW + j] * sm.w2[c * d.LW + j];
    v = wsum(v);
    if (lane == 0) sm.z[s * 16 + c] = v + sm.b2[c];
  }
  __syncthreads();
  // ---- log-softmax + NLL ------------------------------------------------------------------------------
  if (tid < SPB) {
    const int s = tid;
    T mx = sm.z[s * 16]; int am = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c) if (sm.z[s * 16 + c] > mx) { mx = sm.z[s * 16 + c]; am = c; }
    T se = 0;
#pragma unroll
    for (int c = 0; c < NCLS; ++c) se += gexp(sm.z[s * 16 + c] - mx);
    const T lse = mx + glog(se);
    const int y = sm.label[s];
    const T ok = (T)sm.valid[s];
    const T loss = ok * (lse - sm.z[s * 16 + y]);
    if (TRAIN) {
#pragma unroll
      for (int c = 0; c < NCLS; ++c)
        sm.dz[s * 16 + c] = ok * inv_bs * (gexp(sm.z[s * 16 + c] - lse) - (c == y ? (T)1 : (T)0));
      sm.red[s] = loss;
    } else if (ok != (T)0) {
      const size_t o = (size_t)l * a.n_val + sm.sidx[s];
      reinterpret_cast<T*>(a.val_loss)[o] = loss;
      a.val_correct[o] = (unsigned char)(am == y);
    }
  }
  __syncthreads();
  if (!TRAIN) return;

  T* gp = reinterpret_cast<T*>(a.grad_part) + ((size_t)l * S + slice) * a.n_pad;
  if (tid == 0) {
    T tot = 0;
#pragma unroll
    for (int s = 0; s < SPB; ++s) tot += sm.red[s];
    a.loss_part[l * S + slice] = (float)(tot * inv_bs);
    if (a.loss_mirror != nullptr) a.loss_mirror[l * S + slice] = (float)(tot * inv_bs);
  }
  // ---- fc2 grads, dh -----------------------------------------------------------------------------------
  for (int o = tid; o < NCLS * d.LW; o += GNT) {
    const int c = o / d.LW, j = o - c * d.LW;
    T v = 0;
#pragma unroll
    for (int s = 0; s < SPB; ++s) v += sm.dz[s * 16 + c] * sm.h[s * d.LW + j];
    gp[a.off_w2 + o] = v;
  }
  if (tid < NCLS) {
    T v = 0;
#pragma unroll
    for (int s = 0; s < SPB; ++s) v += sm.dz[s * 16 + tid];
    gp[a.off_b2 + tid] = v;
  }
  for (int o = tid; o < SPB * d.LW; o += GNT) {
    const int s = o / d.LW, j = o - s * d.LW;
    T v = 0;
#pragma unroll
    for (int c = 0; c < NCLS; ++c) v += sm.dz[s * 16 + c] * sm.w2[c * d.LW + j];
    sm.dh[o] = sm.h[o] > (T)0 ? v : (T)0;
  }
  __syncthreads();
  if (tid < d.LW) {
    T v = 0;
#pragma unroll
    for (int s = 0; s < SPB; ++s) v += sm.dh[s * d.LW + tid];
    gp[a.off_b1 + tid] = v;
  }
  // ---- da1[s][k] = relu'(a1) sum_j dh[s][j] W1[j][k]: thread per k, coalesced rows of W1 ----------------
  for (int k = tid; k < d.K1; k += GNT) {
    T acc[SPB];
#pragma unroll
    for (int s = 0; s < SPB; ++s) acc[s] = 0;
    for (int j0 = 0; j0 < d.LW; j0 += 8) {
      T wv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) wv[u] = (j0 + u < d.LW) ? ldg(w1 + (size_t)(j0 + u) * d.K1 + k) : (T)0;
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (j0 + u < d.LW) {
#pragma unroll
          for (int s = 0; s < SPB; ++s) acc[s] += sm.dh[s * d.LW + j0 + u] * wv[u];
        }
    }
#pragma unroll
    for (int s = 0; s < SPB; ++s) sm.da1[s * d.K1 + k] = sm.a1[s * d.K1 + k] > (T)0 ? acc[s] : (T)0;
  }
  // ---- dW1[j][k] = sum_s dh[s][j] a1[s][k]: coalesced write-out of the slice's partial ------------------
  for (int j = 0; j < d.LW; ++j) {
    T dj[SPB];
#pragma unroll
    for (int s = 0; s < SPB; ++s) dj[s] = sm.dh[s * d.LW + j];
    T* out = gp + a.off_w1 + (size_t)j * d.K1;
    for (int k = tid; k < d.K1; k += GNT) {
      T v = 0;
#pragma unroll
      for (int s = 0; s < SPB; ++s) v += dj[s] * sm.a1[s * d.K1 + k];
      out[k] = v;
    }
  }
  __syncthreads();
  // ---- conv grads: cells routed through the argmax positions.  Work item = (cell partition q, filter tap or bias):
  //      consecutive threads hold consecutive taps of the same partition, so the da1 / argmax reads are broadcasts ----
  const int ntap = d.F * KS * KS, nitem = ntap + d.F;
  const int npart = max(1, (2 * GNT) / nitem);
  for (int it = tid; it < nitem * npart; it += GNT) {
    const int q = it / nitem, ti = it - q * nitem;
    const bool bias = ti >= ntap;
    const int c = bias ? ti - ntap : ti / (KS * KS);
    const int t = bias ? 0 : ti - c * KS * KS;
    const int ky = t / KS, kx = t - ky * KS;
    const int p0 = (q * d.NP) / npart, p1 = ((q + 1) * d.NP) / npart;
    T acc = 0;
    for (int s = 0; s < SPB; ++s) {
      const T* g = sm.da1 + s * d.K1 + c * d.NP;
      const unsigned char* ag = sm.arg + s * d.K1 + c * d.NP;
      const T* x = sm.img + s * 784 + ky * HW + kx;
      for (int p = p0; p < p1; ++p) {
        const T gv = g[p];
        if (gv != (T)0) {
          if (bias) acc += gv;
          else {
            const int ai = ag[p], py = p / d.PO, px = p - py * d.PO;
            acc += gv * x[(2 * py + (ai >> 1)) * HW + 2 * px + (ai & 1)];
          }
        }
      }
    }
    sm.part[it] = acc;
  }
  __syncthreads();
  if (tid < nitem) {
    T acc = 0;
    for (int q = 0; q < npart; ++q) acc += sm.part[q * nitem + tid];
    gp[tid >= ntap ? a.off_bc + (tid - ntap) : a.off_wc + tid] = acc;
  }
}

template <typename T, int SPB>
NNDT_DEVINL void stage_small(Carve<T, SPB>& sm, const Args& a, const Dims& d, const T* th, int tid) {
  const int ntap = d.F * d.KS * d.KS;
  for (int o = tid; o < ntap; o += GNT) sm.wc[o] = ldg(th + a.off_wc + o);
  for (int o = tid; o < d.F; o += GNT) sm.wc[ntap + o] = ldg(th + a.off_bc + o);
  for (int o = tid; o < d.LW; o += GNT) sm.b1[o] = ldg(th + a.off_b1 + o);
  for (int o = tid; o < NCLS; o += GNT) sm.b2[o] = ldg(th + a.off_b2 + o);
  for (int o = tid; o < NCLS * d.LW; o += GNT) sm.w2[o] = ldg(th + a.off_w2 + o);
}

template <typename T, int KS, int SPB, bool TRAIN>
__global__ void __launch_bounds__(GNT) convnet_generic_kernel(const Args a, const GenericShape gs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Dims d = make_dims(gs);
  Carve<T, SPB> sm(smem_raw, d);
  const int tid = threadIdx.x, l = blockIdx.y;
  pdl_wait();
  pdl_launch_dependents();
  const T* th = reinterpret_cast<const T*>(a.theta) + (size_t)l * a.n_pad;
  stage_small<T, SPB>(sm, a, d, th, tid);
  if (TRAIN) {
    const int call = a.calls != nullptr ? a.calls[l] : 0;
    const BatchGeom bg = batch_geom<true>(a, l, call);
    if (tid < SPB) {
      int idx = 0, lab = 0; float ok = 0.f;
      const uint32_t t = blockIdx.x * SPB + tid;
      if (t < bg.bs) {
        ok = 1.f;
        idx = a.direct ? (int)(l * a.batch + t) : bg.shard_off + (int)feistel_permute(bg.start + t, bg.m, bg.key);
        lab = (int)a.y[idx];
      }
      sm.sidx[tid] = idx; sm.valid[tid] = ok; sm.label[tid] = lab;
    }
    if (tid == 0 && a.calls != nullptr && a.arrive != nullptr) {
      // the last CTA of the node to get here (all have read the counter) advances it
      if (atomicAdd(a.arrive + l, 1u) == gridDim.x - 1) { a.arrive[l] = 0; a.calls[l] = call + 1; }
    }
    __syncthreads();
    generic_chunk<T, KS, SPB, true>(sm, a, d, th, l, blockIdx.x, gridDim.x, (T)1 / (T)(bg.bs ? bg.bs : 1), tid);
  } else {
    const int n_chunks = (a.n_val + SPB - 1) / SPB;
    for (int chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
      __syncthreads();
      if (tid < SPB) {
        const int t = chunk * SPB + tid;
        const bool ok = t < a.n_val;
        sm.sidx[tid] = ok ? t : 0; sm.valid[tid] = ok ? 1.f : 0.f; sm.label[tid] = ok ? (int)a.y[t] : 0;
      }
      __syncthreads();
      generic_chunk<T, KS, SPB, false>(sm, a, d, th, l, 0, 1, (T)1, tid);
    }
  }
}

template <typename T, int KS, int SPB, bool TRAIN>
cudaError_t launch_k(const Args& a, const GenericShape& gs, dim3 grid, cudaStream_t st) {
  const Dims d = make_dims(gs);
  const size_t smem = Carve<T, SPB>::bytes(d);
  auto kern = convnet_generic_kernel<T, KS, SPB, TRAIN>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  return launch_pdl(kern, grid, dim3(GNT), smem, st, a, gs);
}

template <typename T, bool TRAIN>
cudaError_t dispatch(const Args& a, const GenericShape& gs, int spb, dim3 grid, cudaStream_t st) {
  if (gs.KS == 5) return spb == 8 ? launch_k<T, 5, 8, TRAIN>(a, gs, grid, st) : launch_k<T, 5, 4, TRAIN>(a, gs, grid, st);
  if (gs.KS == 3) return spb == 8 ? launch_k<T, 3, 8, TRAIN>(a, gs, grid, st) : launch_k<T, 3, 4, TRAIN>(a, gs, grid, st);
  return cudaErrorInvalidValue;
}

}  // namespace

size_t generic_smem_bytes(const GenericShape& gs, int dtype64, int spb) {
  const Dims d = make_dims(gs);
  if (dtype64) return spb == 8 ? Carve<double, 8>::bytes(d) : Carve<double, 4>::bytes(d);
  return spb == 8 ? Carve<float, 8>::bytes(d) : Carve<float, 4>::bytes(d);
}

cudaError_t launch_generic_train(const Args& a, const GenericShape& gs, int spb, int S, cudaStream_t st) {
  const dim3 grid(S, a.L);
  return gs.dtype64 ? dispatch<double, true>(a, gs, spb, grid, st) : dispatch<float, true>(a, gs, spb, grid, st);
}

int generic_eval_spb(const GenericShape& gs) {
  return generic_smem_bytes(gs, gs.dtype64, 8) <= 160 * 1024 ? 8 : 4;
}

cudaError_t launch_generic_eval(const Args& a, const GenericShape& gs, int ctas_per_node, cudaStream_t st) {
  const dim3 grid(ctas_per_node, a.L);
  const int spb = generic_eval_spb(gs);
  return gs.dtype64 ? dispatch<double, false>(a, gs, spb, grid, st) : dispatch<float, false>(a, gs, spb, grid, st);
}

}  // namespace mnist
}  // namespace nndt
