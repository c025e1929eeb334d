// float64 training and evaluation kernels of the implicit-density MLPs (FourierNet / FFReLUNet [2, H1, 64, 64, 64, 1],
// H1 in {64, 128, 256}) for sm_90a: the reference's precision (models/fourier_nn.py sets float64 as the default tensor
// type).  Every contraction runs on the FP64 tensor cores as warp-level mma.sync m16n8k4 (DMMA) with fp64
// accumulation; the SIREN layer uses full-precision sin / sincos, the sigmoid, log and the loss are fp64.
//
// Decomposition: one 2-CTA thread-block cluster per tile of TR = 32 batch rows, layer 1 split by its H1 features.
//   * CTA r owns the features [r H1/2, (r+1) H1/2): its slices of W0 / b0, of h1 (all 32 rows) and of W1's columns,
//     and computes the partial layer-2 pre-activation z2_r = h1_r . W1_r^T of all 32 rows.
//   * The pair reduce-scatters z2 by rows over distributed shared memory: CTA r finishes rows [16 r, 16 r + 16) and
//     runs layers 2-5, the loss and the backward down to dz2 on them (W2 and W3 are resident in both CTAs).
//   * dz2 is all-gathered back to both CTAs; dW1_r = dz2^T . h1_r, dz1_r = (dz2 . W1_r) * act'(z1_r) and the
//     first-layer gradients need no further cross-CTA traffic.
// Shared memory per CTA (sizeof(Smem<H1>); every row is padded by 4 doubles, so fragment reads, row-wise or transposed,
// are free of bank conflicts):
//                              H1 = 64    128      256
//   W1 slice [64][H1/2 + 4]     18.0 KB   34.0 KB  66.0 KB
//   W2, W3 [64][68]             68.0 KB   68.0 KB  68.0 KB
//   h1 / dz1 [32][H1/2 + 4]      9.0 KB   17.0 KB  33.0 KB
//   partial z2 / dz2 [32][68]   17.0 KB   17.0 KB  17.0 KB
//   h2, h3, h4 / dz4 [16][68]   25.5 KB   25.5 KB  25.5 KB
//   vectors and accumulators     6.6 KB    8.1 KB  11.1 KB
//   total                      144.1 KB  169.6 KB 220.6 KB   (limit 227 KB)
// Weight gradients accumulate over all tiles of a node in registers, as the DMMA accumulators of dW1_r, dW2 and dW3;
// bias, w4 and W0 gradients in shared memory, each element owned by one thread.  Every reduction runs in a fixed order
// and nothing is added atomically, so two launches on the same inputs give bitwise-equal gradients and losses.
#include "common.cuh"
#include "mlp.h"
#include "sampler.cuh"

namespace nndt {
namespace mlp {
namespace f64 {

constexpr int NT = 256;          // 8 warps per CTA
constexpr int TR = 32;           // rows of a cluster tile
constexpr int OR = 16;           // rows a CTA owns for layers 2-5 (TR / 2)
constexpr int HID = 64;
constexpr int PAD = 4;           // row strides = 4 mod 16 doubles: the 16 lanes of a half-warp hit 16 distinct bank pairs
constexpr int HS = HID + PAD;

template <int H1>
struct Smem {
  static constexpr int HF = H1 / 2, FS = HF + PAD;
  double w1[HID * FS];           // W1[o][r HF + f]
  double w2[HID * HS];
  double w3[HID * HS];
  double h1[TR * FS];            // h1 of the tile's rows, own features; later dz1
  double zp[TR * HS];            // partial z2 of the tile's rows; later dz2 of the tile's rows
  double h2[OR * HS];            // own rows: h2
  double h3[OR * HS];            // own rows: h3, later dz3
  double h4[OR * HS];            // own rows: h4, later dz4
  double w0[HF * 2], b0[HF];
  double b1[HID], b2[HID], b3[HID], w4[HID];
  double xs[TR * 2], ys[TR];
  double dz5[OR], lrow[OR];
  double g_w0[HF * 2], g_b0[HF];
  double g_b1[HID], g_b2[HID], g_b3[HID], g_w4[HID];
  double b4, g_b4, g_loss;
  int ridx[TR];
};
static_assert(sizeof(Smem<256>) <= 227 * 1024, "shared memory budget");

// ---- shared stages ------------------------------------------------------------------------------------------------
template <int H1>
NNDT_DEVINL void stage_weights(Smem<H1>& sm, const Args& a, const double* th, int rank, int tid) {
  constexpr int HF = Smem<H1>::HF, FS = Smem<H1>::FS;
  for (int e = tid; e < HID * HF; e += NT) {
    const int o = e / HF, f = e - o * HF;
    sm.w1[o * FS + f] = th[a.off[2] + o * H1 + rank * HF + f];
  }
  for (int e = tid; e < HID * HID; e += NT) {
    const int o = e / HID, i = e - o * HID;
    sm.w2[o * HS + i] = th[a.off[4] + e];
    sm.w3[o * HS + i] = th[a.off[6] + e];
  }
  for (int e = tid; e < HF * 2; e += NT) sm.w0[e] = th[a.off[0] + rank * HF * 2 + e];
  for (int e = tid; e < HF; e += NT) sm.b0[e] = th[a.off[1] + rank * HF + e];
  if (tid < HID) {
    sm.b1[tid] = th[a.off[3] + tid];
    sm.b2[tid] = th[a.off[5] + tid];
    sm.b3[tid] = th[a.off[7] + tid];
    sm.w4[tid] = th[a.off[8] + tid];
  }
  if (tid == 0) sm.b4 = th[a.off[9]];
}

// first-layer pre-activation of row r, own feature f
template <int H1>
NNDT_DEVINL double z1(const Smem<H1>& sm, int r, int f) {
  return fma(sm.xs[2 * r + 1], sm.w0[2 * f + 1], fma(sm.xs[2 * r], sm.w0[2 * f], sm.b0[f]));
}

// dst[r][n] = relu(src[r] . W[n] + b[n]) for the 16 own rows; warp w computes columns 8 w .. 8 w + 7
NNDT_DEVINL void hidden_layer(const double* src, const double* w, const double* b, double* dst, int warp, int lane) {
  double c[1][4];
  zero(c);
  gemm<1>(c, 0, 8 * warp, HID, lane, at(src, HS), at_t(w, HS));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = frow(0, lane, i), n = fcol(8 * warp, lane, i);
    dst[r * HS + n] = fmax(c[0][i] + b[n], 0.0);
  }
}

// Layers 1-4 of the tile whose 32 inputs are in sm.xs: h4 of the own rows in sm.h4.  The cluster barrier inside makes
// both CTAs' partial z2 visible; the peer reads this CTA's zp rows of its half until its next cluster barrier.
template <int H1>
NNDT_DEVINL void forward_tile(Smem<H1>& sm, const Args& a, int rank, int tid) {
  constexpr int HF = Smem<H1>::HF, FS = Smem<H1>::FS;
  const int warp = tid >> 5, lane = tid & 31;
  for (int e = tid; e < TR * HF; e += NT) {
    const int r = e / HF, f = e - r * HF;
    const double z = z1(sm, r, f);
    sm.h1[r * FS + f] = fmax(a.first_act == kFirstSinRelu ? sin(a.scale64 * z) : z, 0.0);
  }
  __syncthreads();
  {
    double c[2][4];
    zero(c);
    const int m0 = 16 * (warp & 1), n0 = 16 * (warp >> 1);
    gemm<2>(c, m0, n0, HF, lane, at(sm.h1, FS), at_t(sm.w1, FS));
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) sm.zp[frow(m0, lane, i) * HS + fcol(n0 + 8 * j, lane, i)] = c[j][i];
  }
  cluster_sync();
  // reduce-scatter: the own rows' z2 = partial(rank 0) + partial(rank 1)
  for (int e = tid; e < OR * HID; e += NT) {
    const int r = e / HID, n = e - r * HID;
    const double* p = &sm.zp[(OR * rank + r) * HS + n];
    const double v = *p + ld_dsmem(map_to(p, (uint32_t)(rank ^ 1)));
    sm.h2[r * HS + n] = fmax(v + sm.b1[n], 0.0);
  }
  __syncthreads();
  hidden_layer(sm.h2, sm.w2, sm.b2, sm.h3, warp, lane);
  __syncthreads();
  hidden_layer(sm.h3, sm.w3, sm.b3, sm.h4, warp, lane);
  __syncthreads();
}

// output pre-activation z5 of own row r (valid in lane 0)
template <int H1>
NNDT_DEVINL double out_layer(const Smem<H1>& sm, int r, int lane) {
  const double d = fma(sm.h4[r * HS + lane], sm.w4[lane], sm.h4[r * HS + lane + 32] * sm.w4[lane + 32]);
  return warp_sum(d) + sm.b4;
}

// ---- forward: out[l][row] for every node l = blockIdx.y, grid-stride over the tiles --------------------------------
template <int H1>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(NT, 1) mlp_f64_forward_kernel(const Args a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem<H1>& sm = *reinterpret_cast<Smem<H1>*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rank = (int)cluster_rank(), l = blockIdx.y;
  const int NC = gridDim.x / 2, c = blockIdx.x / 2;
  const double* x = reinterpret_cast<const double*>(a.x);
  double* out = reinterpret_cast<double*>(a.out) + (size_t)l * a.n_rows;
  stage_weights(sm, a, reinterpret_cast<const double*>(a.theta) + (size_t)l * a.n_pad, rank, tid);
  const int ntiles = (a.n_rows + TR - 1) / TR;
  for (int tile = c; tile < ntiles; tile += NC) {
    const int row0 = tile * TR;
    if (tid < TR * 2) sm.xs[tid] = row0 + (tid >> 1) < a.n_rows ? x[(size_t)row0 * 2 + tid] : 0.0;
    __syncthreads();
    forward_tile(sm, a, rank, tid);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = 2 * warp + h, row = row0 + OR * rank + r;
      const double z = out_layer(sm, r, lane);
      if (lane == 0 && row < a.n_rows) out[row] = a.last_act == kLastSigmoid ? 1.0 / (1.0 + exp(-z)) : z;
    }
    cluster_sync();      // the peer has read this tile's partial z2 before the next tile overwrites it
  }
}

// ---- training: one minibatch per node, gradients to per-CTA partial rows ------------------------------------------
// Static partition of the items (node, tile) in node-major order over the clusters; CTA r of the c-th cluster that
// covers node l owns slot 2 c + r of the node's partial rows and writes all of it once, after the node's last tile:
// its share of every gradient, zeros in the peer's W0 / b0 / W1 columns.  Clusters never wait on each other, so every
// cluster count is a valid launch.
template <int H1>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(NT, 1) mlp_f64_train_kernel(const Args a) {
  constexpr int HF = Smem<H1>::HF, FS = Smem<H1>::FS;
  constexpr int NJ1 = HF / 16, NJZ = HF / 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem<H1>& sm = *reinterpret_cast<Smem<H1>*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rank = (int)cluster_rank();
  const uint32_t peer = (uint32_t)(rank ^ 1);
  const double* x = reinterpret_cast<const double*>(a.x);
  const double* y = reinterpret_cast<const double*>(a.y);
  double* grad_part = reinterpret_cast<double*>(a.grad_part);
  double* loss_part = reinterpret_cast<double*>(a.loss_part);

  const int Tmax = (a.batch + TR - 1) / TR;
  const int I = a.L * Tmax, NC = gridDim.x / 2, c = blockIdx.x / 2;
  const int it0 = (int)(((long long)c * I) / NC), it1 = (int)(((long long)(c + 1) * I) / NC);

  // weight-gradient accumulators: dW1 rows 16 (w & 3) .. + 16, own columns (HF / 2) (w >> 2) .. + HF / 2;
  // dW2 and dW3 rows 16 (w & 3) .. + 16, columns 32 (w >> 2) .. + 32
  const int gm0 = 16 * (warp & 3);
  const int g1n0 = (HF / 2) * (warp >> 2), g2n0 = 32 * (warp >> 2);
  double acc1[NJ1][4], acc2[4][4], acc3[4][4];
  int cur = -1, slot = 0;
  NodeStream ns{};

  auto flush = [&]() {
    double* gp = grad_part + ((size_t)cur * a.S + slot) * a.n_pad;
#pragma unroll
    for (int j = 0; j < NJ1; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i)
        gp[a.off[2] + frow(gm0, lane, i) * H1 + rank * HF + fcol(g1n0 + 8 * j, lane, i)] = acc1[j][i];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int o = frow(gm0, lane, i), n = fcol(g2n0 + 8 * j, lane, i);
        gp[a.off[4] + o * HID + n] = acc2[j][i];
        gp[a.off[6] + o * HID + n] = acc3[j][i];
      }
    for (int e = tid; e < HID * HF; e += NT) {
      const int o = e / HF, f = e - o * HF;
      gp[a.off[2] + o * H1 + (rank ^ 1) * HF + f] = 0.0;
    }
    for (int e = tid; e < H1 * 2; e += NT) {
      const int own = e - rank * HF * 2;
      gp[a.off[0] + e] = (own >= 0 && own < HF * 2) ? sm.g_w0[own] : 0.0;
    }
    for (int e = tid; e < H1; e += NT) {
      const int own = e - rank * HF;
      gp[a.off[1] + e] = (own >= 0 && own < HF) ? sm.g_b0[own] : 0.0;
    }
    if (tid < HID) {
      gp[a.off[3] + tid] = sm.g_b1[tid];
      gp[a.off[5] + tid] = sm.g_b2[tid];
      gp[a.off[7] + tid] = sm.g_b3[tid];
      gp[a.off[8] + tid] = sm.g_w4[tid];
    }
    if (tid == 0) {
      gp[a.off[9]] = sm.g_b4;
      loss_part[cur * a.S + slot] = sm.g_loss / (double)ns.size;
    }
  };

  for (int it = it0; it < it1; ++it) {
    const int l = it / Tmax;
    if (l != cur) {
      if (cur >= 0) {
        flush();
        __syncthreads();
      }
      cur = l;
      {
        const long long first_item = (long long)l * Tmax;
        int cf = (int)((first_item * NC) / I);
        while ((long long)(cf + 1) * I / NC <= first_item) ++cf;
        while ((long long)cf * I / NC > first_item) --cf;
        slot = 2 * (c - cf) + rank;
      }
      stage_weights(sm, a, reinterpret_cast<const double*>(a.theta) + (size_t)l * a.n_pad, rank, tid);
      zero(acc1); zero(acc2); zero(acc3);
      for (int e = tid; e < HF * 2; e += NT) sm.g_w0[e] = 0.0;
      for (int e = tid; e < HF; e += NT) sm.g_b0[e] = 0.0;
      if (tid < HID) sm.g_b1[tid] = sm.g_b2[tid] = sm.g_b3[tid] = sm.g_w4[tid] = 0.0;
      if (tid == 0) sm.g_b4 = sm.g_loss = 0.0;
      const long long* wt = a.win_table != nullptr
                                ? reinterpret_cast<const long long*>(a.win_table) + (size_t)l * kWinTableLen : nullptr;
      ns = node_stream((uint32_t)a.calls[l], (uint32_t)a.shard_len[l], (uint32_t)a.batch, (uint32_t)a.seed,
                       (uint32_t)(a.node0 + l), a.shard_off[l], wt);
      __syncthreads();
    }
    const uint32_t t0 = (uint32_t)(it - l * Tmax) * TR;
    if (t0 >= ns.size) continue;                         // partial batch: nothing in this tile (the same in both CTAs)
    const double bs = (double)ns.size;

    // ---- gather the tile's rows (both CTAs draw all 32) ----------------------------------------------------------
    if (tid < TR) {
      const int idx = t0 + tid < ns.size ? stream_row(ns, t0 + tid) : -1;
      sm.ridx[tid] = idx;
      sm.ys[tid] = idx >= 0 ? y[idx] : 0.0;
      sm.xs[2 * tid] = idx >= 0 ? x[(size_t)idx * 2] : 0.0;
      sm.xs[2 * tid + 1] = idx >= 0 ? x[(size_t)idx * 2 + 1] : 0.0;
    }
    __syncthreads();
    forward_tile(sm, a, rank, tid);

    // ---- output layer, loss, dL/dz5 of the own rows ----------------------------------------------------------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = 2 * warp + h;
      const double z = out_layer(sm, r, lane);
      if (lane == 0) {
        const bool valid = sm.ridx[OR * rank + r] >= 0;
        const double yv = sm.ys[OR * rank + r];
        double p = z, dpdz = 1.0;
        if (a.last_act == kLastSigmoid) { p = 1.0 / (1.0 + exp(-z)); dpdz = p * (1.0 - p); }
        double loss, gz;
        if (a.loss == kLossBCE) {
          // torch.nn.BCELoss clamps the logs at -100.  With the sigmoid, dL/dz = p - y: the derivative of the exact
          // loss, which equals torch's (p - y) / max(p (1 - p), 1e-12) * p (1 - p) wherever p (1 - p) > 1e-12; on
          // saturated rows torch's gradient shrinks with p (1 - p), this one does not.
          loss = -(yv * fmax(log(p), -100.0) + (1.0 - yv) * fmax(log(1.0 - p), -100.0));
          gz = (a.last_act == kLastSigmoid) ? (p - yv) : (p - yv) / fmax(p * (1.0 - p), 1e-12);
        } else if (a.loss == kLossMSE) {
          loss = (p - yv) * (p - yv); gz = 2.0 * (p - yv) * dpdz;
        } else {
          loss = fabs(p - yv); gz = (p > yv ? 1.0 : (p < yv ? -1.0 : 0.0)) * dpdz;
        }
        sm.dz5[r] = valid ? gz / bs : 0.0;
        sm.lrow[r] = valid ? loss : 0.0;
      }
    }
    __syncthreads();

    // ======================= backward ===============================================================================
    // layer 5: dW4 += dz5^T h4, db4 += sum dz5, dz4 = dz5 w4 relu'(h4) over h4, db3 += sum dz4; one thread per column
    if (tid < HID) {
      double gw = 0.0, gb = 0.0;
      for (int r = 0; r < OR; ++r) {
        const double hv = sm.h4[r * HS + tid], d5 = sm.dz5[r];
        gw = fma(d5, hv, gw);
        const double d4 = hv > 0.0 ? d5 * sm.w4[tid] : 0.0;
        sm.h4[r * HS + tid] = d4;
        gb += d4;
      }
      sm.g_w4[tid] += gw;
      sm.g_b3[tid] += gb;
    } else if (tid == HID) {
      double ls = 0.0, gb = 0.0;
      for (int r = 0; r < OR; ++r) { ls += sm.lrow[r]; gb += sm.dz5[r]; }
      sm.g_loss += ls;
      sm.g_b4 += gb;
    }
    __syncthreads();
    // layer 4: dW3 += dz4^T h3; dz3 = (dz4 . W3) relu'(h3) over h3
    {
      gemm<4>(acc3, gm0, g2n0, OR, lane, at_t(sm.h4, HS), at(sm.h3, HS));
      double d[1][4];
      zero(d);
      gemm<1>(d, 0, 8 * warp, HID, lane, at(sm.h4, HS), at(sm.w3, HS));
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        double* p = &sm.h3[frow(0, lane, i) * HS + fcol(8 * warp, lane, i)];
        *p = *p > 0.0 ? d[0][i] : 0.0;
      }
      __syncthreads();
    }
    // layer 3: db2 += sum dz3; dW2 += dz3^T h2; dz2 = (dz3 . W2) relu'(h2) to the own rows of both CTAs' zp
    {
      if (tid < HID) {
        double gb = 0.0;
        for (int r = 0; r < OR; ++r) gb += sm.h3[r * HS + tid];
        sm.g_b2[tid] += gb;
      }
      gemm<4>(acc2, gm0, g2n0, OR, lane, at_t(sm.h3, HS), at(sm.h2, HS));
      double d[1][4];
      zero(d);
      gemm<1>(d, 0, 8 * warp, HID, lane, at(sm.h3, HS), at(sm.w2, HS));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = frow(0, lane, i), n = fcol(8 * warp, lane, i);
        const double v = sm.h2[r * HS + n] > 0.0 ? d[0][i] : 0.0;
        double* p = &sm.zp[(OR * rank + r) * HS + n];
        *p = v;
        st_dsmem(map_to(p, peer), v);
      }
      cluster_sync();                                    // dz2 of all 32 rows is in both CTAs
    }
    // layer 2: db1 += sum dz2 (own rows); dW1_r += dz2^T h1_r (all rows)
    if (tid < HID) {
      double gb = 0.0;
      for (int r = 0; r < OR; ++r) gb += sm.zp[(OR * rank + r) * HS + tid];
      sm.g_b1[tid] += gb;
    }
    gemm<NJ1>(acc1, gm0, g1n0, TR, lane, at_t(sm.zp, HS), at(sm.h1, FS));
    __syncthreads();                                     // h1 is dead: dz1 goes over it
    // layer 1: dz1_r = (dz2 . W1_r) act'(z1); one 16 x 8 tile at a time, which keeps the sincos of the epilogue
    // clear of the accumulators' registers
    const int zm0 = 16 * (warp & 1), zn0 = (HF / 4) * (warp >> 1);
#pragma unroll 1
    for (int j = 0; j < NJZ; ++j) {
      double d[1][4];
      zero(d);
      gemm<1>(d, zm0, zn0 + 8 * j, HID, lane, at(sm.zp, HS), at(sm.w1, FS));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = frow(zm0, lane, i), f = fcol(zn0 + 8 * j, lane, i);
        const double z = z1(sm, r, f);
        double dact;
        if (a.first_act == kFirstSinRelu) {
          double sn, cs;
          sincos(a.scale64 * z, &sn, &cs);
          dact = sn > 0.0 ? cs * a.scale64 : 0.0;
        } else {
          dact = z > 0.0 ? 1.0 : 0.0;
        }
        sm.h1[r * FS + f] = d[0][i] * dact;
      }
    }
    __syncthreads();
    // [dW0 | db0]_r += dz1_r^T [x, 1]; one thread per own feature
    if (tid < HF) {
      double g0 = 0.0, g1 = 0.0, gb = 0.0;
      for (int r = 0; r < TR; ++r) {
        const double d1 = sm.h1[r * FS + tid];
        g0 = fma(d1, sm.xs[2 * r], g0);
        g1 = fma(d1, sm.xs[2 * r + 1], g1);
        gb += d1;
      }
      sm.g_w0[2 * tid] += g0;
      sm.g_w0[2 * tid + 1] += g1;
      sm.g_b0[tid] += gb;
    }
    __syncthreads();                                     // the next tile overwrites xs / h1 / zp
  }
  if (cur >= 0) flush();
  // no distributed-shared-memory access follows the last cluster barrier: the CTAs may exit independently
}

template <int H1>
static cudaError_t launch_forward_t(const Args& a, int clusters, cudaStream_t st) {
  const int smem = (int)sizeof(Smem<H1>);
  static cudaError_t attr = cudaFuncSetAttribute(mlp_f64_forward_kernel<H1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (attr != cudaSuccess) return attr;
  mlp_f64_forward_kernel<H1><<<dim3(2 * clusters, a.L), NT, smem, st>>>(a);
  return cudaGetLastError();
}

template <int H1>
static cudaError_t launch_train_t(const Args& a, int clusters, cudaStream_t st) {
  const int smem = (int)sizeof(Smem<H1>);
  static cudaError_t attr = cudaFuncSetAttribute(mlp_f64_train_kernel<H1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (attr != cudaSuccess) return attr;
  mlp_f64_train_kernel<H1><<<dim3(2 * clusters), NT, smem, st>>>(a);
  return cudaGetLastError();
}

template <int H1>
static int max_clusters_t() {
  const int smem = (int)sizeof(Smem<H1>);
  if (cudaFuncSetAttribute(mlp_f64_train_kernel<H1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2, 1, 1); cfg.blockDim = dim3(NT); cfg.dynamicSmemBytes = smem;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, mlp_f64_train_kernel<H1>, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

}  // namespace f64

cudaError_t launch_forward_f64(const Args& a, int clusters_per_node, cudaStream_t st) {
  if (a.d_in != 2 || clusters_per_node < 1) return cudaErrorInvalidValue;
  switch (a.h1) {
    case 64: return f64::launch_forward_t<64>(a, clusters_per_node, st);
    case 128: return f64::launch_forward_t<128>(a, clusters_per_node, st);
    case 256: return f64::launch_forward_t<256>(a, clusters_per_node, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_train_f64(const Args& a, int clusters, cudaStream_t st) {
  // no `direct` mode: the density problems always sample in the kernel
  if (a.d_in != 2 || a.direct || clusters < 1) return cudaErrorInvalidValue;
  switch (a.h1) {
    case 64: return f64::launch_train_t<64>(a, clusters, st);
    case 128: return f64::launch_train_t<128>(a, clusters, st);
    case 256: return f64::launch_train_t<256>(a, clusters, st);
    default: return cudaErrorInvalidValue;
  }
}

int f64_max_active_clusters(int h1) {
  switch (h1) {
    case 64: return f64::max_clusters_t<64>();
    case 128: return f64::max_clusters_t<128>();
    case 256: return f64::max_clusters_t<256>();
    default: return 0;
  }
}

}  // namespace mlp
}  // namespace nndt
