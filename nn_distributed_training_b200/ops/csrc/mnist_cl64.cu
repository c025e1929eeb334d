// float64 training kernel of the paper's MNISTConvNet(3, 5, 64) at batch <= 64: a K-split thread-block-cluster
// decomposition with the three fc1-sized contractions on the FP64 tensor cores (mma.sync m16n8k4, DMMA, fp64
// accumulation) and the conv layer on the fp64 CUDA cores.  This is the kernel behind the framework's float64 arm — the
// precision the reference runs end to end (experiments/dist_mnist_ex.py:19) — and replaces the batch-split generic
// kernel (mnist_generic.cu) there, which streams the 221 KB fp64 W1 matrix three times per CTA.
//
// A node is `nsplit` clusters of 4 CTAs (MS = 64 / nsplit samples each); CTA c owns pooled rows {3c, 3c+1, 3c+2} of all
// three channels = 108 of the 432 fc1 inputs for all MS samples (image rows 6c .. 6c+9): conv+ReLU+pool -> A_c [MS x 108];
// H_c = A_c . W1_c^T reduced over the cluster through distributed shared memory (reduce-scatter by samples, MS / 4 per
// CTA; fc2 / loss / backward on the owners, dH rows gathered back); da1_c = dH . W1_c and dW1_c = dH^T . A_c are local;
// dW1_c goes straight to its columns of the gradient row; small gradients are reduced through DSMEM.  At MS <= 32 the
// partial H, dH and the small-gradient shares are pushed (st.async) on transaction barriers instead of read between
// cluster barriers.  One gradient partial row per cluster.
// Why 4 CTAs: a cluster must sit inside one GPC and a CTA fills its SM (shared memory and registers), so a GPC of n SMs
// holds floor(n / CL) clusters.  On an H100 SXM (132 SMs) only 17 six-CTA clusters fit at once, and the 20 clusters of
// 10 nodes x 2 batch splits ran in two waves; 4-CTA clusters keep every node count up to 12 in one wave.
// Row strides are 4 mod 16 doubles (116, 68), so DMMA fragment reads, row-wise or transposed, are free of bank
// conflicts.  Every sum runs in a fixed order and nothing is added atomically: two launches on the same inputs give
// bitwise-equal gradients and losses.
#include "mnist_device.cuh"

namespace nndt {
namespace mnist {

namespace cl64 {

// 20 warps of 96 registers a thread (61,440 of the SM's 65,536): the forward conv takes fewer rounds than at 16 warps,
// and GEMM 3 gets four warps of its own beside the 15 conv-gradient warps and the bias warp
constexpr int NT = 640, CL = 4, CELLS = 36, KC = 108, WS = 116, HS = 68;
constexpr int PXR = 10 * HW;                  // image rows 6c .. 6c+9 of a sample: 280 pixels
constexpr int KT = (KC + 7) / 8;              // 8-column tiles over a CTA's fc1 inputs; columns 108..111 fall in the row padding
// rows of w2 and of the owners' h hold the 64 hidden units as four 16-unit runs 17 apart: the fc2 logits are summed by
// 4 lanes per class over one run each, and with runs 17 apart (class rows 68 = 4 mod 16) the 32 lanes of a warp read
// every 8-byte bank twice instead of all hitting one
constexpr int HR = 68;
NNDT_DEVINL int hr(int j) { return (j >> 4) * 17 + (j & 15); }
constexpr int PART_WC = 0, PART_BC = 75, PART_B1 = 78, PART_W2 = 142, PART_B2 = 782, PART_LOSS = 792, PART_N = 793;

template <int MS>
struct Smem {
  static constexpr int NO = MS / CL;           // samples a CTA owns for fc2, the loss and their backward
  // MS <= 32: partial H, dH and the fc2 / b1 / b2 / loss shares cross CTAs as pushes (st.async) into receive buffers,
  // each counted on the receiver's transaction barrier.  MS = 64 has no room for the buffers and keeps the
  // cluster-barrier path: its owners' partial H and dH rows are read by the peers (ld.shared::cluster)
  static constexpr bool kPush = MS <= 32;
  static constexpr int PER = (PART_N - PART_B1 + CL - 1) / CL;   // fc2 / b1 / b2 / loss entries each CTA reduces
  static constexpr bool kDoublePix = MS <= 32; // pixels as normalised doubles; at MS = 64 they only fit as raw bytes
  // sample stride of the pixel rows; as doubles 282 (141 16-byte units, odd), so the same patch row of eight consecutive
  // samples starts in eight different 16-byte bank groups
  static constexpr int PXS = kDoublePix ? PXR + 2 : PXR;
  double w[HID * WS];        // W1 slice [j][k], k = ch * 36 + cell; after GEMM 2 da1 [k][s], then the conv-grad warp sums
  double a[MS * WS];         // A tile [s][k]
  // kPush: dH [s][j], pushed by the owners.  Otherwise partial H [s][j] (read by the peers), after barrier #2 dH [s][j]
  alignas(16) double h[MS * HS];
  alignas(16) unsigned char img[kDoublePix ? MS * PXS * 8 : MS * PXS];
  double lut[kDoublePix ? 1 : 256];                         // MS = 64: normalised value of each u8 pixel
  double h_loc[NO * HR > CL * 80 ? NO * HR : CL * 80];     // [sl][hr(j)]; later (rank 0) the conv-gradient shares [CL][80]
  double dh_loc[NO * HID];
  double part[800];
  double w2[NCLS * HR];                                     // [cc][hr(j)]
  alignas(16) double b1[HID];                               // b1, b2 arrive by 16-byte cp.async with the W1 slice
  alignas(16) double b2[16];
  double wc[80];
  double dz[NO * 16];
  double red[NO];
  int sidx[MS];
  int label[MS];
  float valid[MS];
  unsigned char arg[MS * KC];
  // kPush receive buffers: [src rank][sl][j] the four partial H of this CTA's samples (later, on rank 0, the conv-gradient
  // shares [CL][80]), and [src rank][PER] the shares of this CTA's quarter of the fc2 / b1 / b2 / loss gradients
  alignas(16) double hin[kPush ? CL * NO * HID : 2];
  double shr[kPush ? CL * PER : 1];
  uint64_t bar[3];           // kPush: H in, dH in, shares in; each completes once per launch (parity 0)
};
static_assert(sizeof(Smem<16>) <= 227 * 1024 && sizeof(Smem<32>) <= 227 * 1024 && sizeof(Smem<64>) <= 227 * 1024,
              "shared memory budget");

NNDT_DEVINL double wmax(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// one exchange step of warp_reduce_scatter16: the lanes with bit 2H set keep the upper half of their H values
template <int H>
NNDT_DEVINL void fold_half(double (&v)[16], int lane) {
  const bool up = (lane & (2 * H)) != 0;
#pragma unroll
  for (int i = 0; i < H; ++i) {
    const double send = up ? v[i] : v[i + H], keep = up ? v[i + H] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2 * H);
  }
}
// Sums v[0 .. 15] over the warp in a fixed order with 16 shuffles instead of 80: every exchange step halves the values a
// lane keeps.  Afterwards lanes 2i and 2i + 1 hold the warp total of v[i] in v[0].
NNDT_DEVINL void warp_reduce_scatter16(double (&v)[16], int lane) {
  fold_half<8>(v, lane); fold_half<4>(v, lane); fold_half<2>(v, lane); fold_half<1>(v, lane);
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
}
// The DMMA k-loop of this kernel: c[j] += sum_k A(m0 + ., k) B(k, n0 + 8 j + .) over k < K, step by step in the k order of
// gemm() in common.cuh, so every accumulator sees the same products in the same sequence.  K is a compile-time constant
// and the loop is unrolled; the fragments of step k + 4 are read before the DMMA of step k, and the mma is not volatile,
// so the compiler may schedule the shared-memory reads of the next step under the current DMMA chain.
NNDT_DEVINL void dmma_nv(double (&c)[4], double a0, double a1, double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a0), "d"(a1), "d"(b));
}
template <int NJ, int K, class FA, class FB>
NNDT_DEVINL void gemm_k(double (&c)[NJ][4], int m0, int n0, int lane, FA A, FB B) {
  static_assert(K % 4 == 0, "k steps of 4");
  const int g = lane >> 2, t = lane & 3;
  double a0 = A(m0 + g, t), a1 = A(m0 + g + 8, t), b[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) b[j] = B(t, n0 + 8 * j + g);
#pragma unroll
  for (int k0 = 0; k0 < K; k0 += 4) {
    double na0 = 0.0, na1 = 0.0, nb[NJ];
    if (k0 + 4 < K) {
      const int k = k0 + 4 + t;
      na0 = A(m0 + g, k); na1 = A(m0 + g + 8, k);
#pragma unroll
      for (int j = 0; j < NJ; ++j) nb[j] = B(k, n0 + 8 * j + g);
    }
#pragma unroll
    for (int j = 0; j < NJ; ++j) dmma_nv(c[j], a0, a1, b[j]);
    if (k0 + 4 < K) {
      a0 = na0; a1 = na1;
#pragma unroll
      for (int j = 0; j < NJ; ++j) b[j] = nb[j];
    }
  }
}
NNDT_DEVINL void stamp(long long* prof, int idx, int tid) {
  if (prof != nullptr && tid == 0) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    prof[idx] = t;
  }
}

template <int MS>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(NT, 1)
mnist_cl64_train_kernel(const Args a, const GenericShape gs) {
  using SM = Smem<MS>;
  constexpr int NO = SM::NO, PXS = SM::PXS;
  constexpr bool kDoublePix = SM::kDoublePix;
  static_assert(MS % 16 == 0 && NO <= NT / 32, "tile geometry");
  static_assert(CELLS % 2 == 0 && NCLS % 2 == 0 && 32 + NCLS / 2 <= NT, "16-byte parameter copies");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int l = blockIdx.z, bsplit = blockIdx.y, nsplit = gridDim.y;
  const int c = (int)cluster_rank();
  const double* th = reinterpret_cast<const double*>(a.theta) + (size_t)l * a.n_pad;
  const double pmean = gs.mean, pis = gs.inv_std;
  const bool u8 = a.x_is_u8 != 0;
  double* imgd = reinterpret_cast<double*>(sm.img);
  // pixel p (0 .. 279) of sample s's image rows 6c .. 6c+9.  fp32 inputs at MS = 64 have no room in shared memory and
  // are read from L2 (the rows were just loaded); invalid samples are masked wherever their pixels would count.
  auto pix = [&](int s, int p) -> double {
    if constexpr (kDoublePix) return imgd[s * PXS + p];
    else if (u8) return sm.lut[sm.img[s * PXR + p]];
    else return (double)__ldg(reinterpret_cast<const float*>(a.x) + (size_t)sm.sidx[s] * 784 + 6 * HW * c + p);
  };
  long long* prof = a.prof != nullptr ? a.prof + ((l * nsplit + bsplit) * CL + c) * 64 : nullptr;
  stamp(prof, 0, tid);
  constexpr bool kPush = SM::kPush;
  constexpr int PER = SM::PER;
  if constexpr (kPush) {
    static_assert(CL * NO * HID >= CL * 80, "rank 0's partial-H buffer holds the conv-gradient shares");
    if (tid == 0) {
      for (int i = 0; i < 3; ++i) mbarrier_init(&sm.bar[i], 1);
      mbarrier_expect_tx(&sm.bar[0], CL * NO * HID * 8);
      mbarrier_expect_tx(&sm.bar[1], MS * HID * 8);
      mbarrier_expect_tx(&sm.bar[2], CL * min(PER, PART_N - PART_B1 - c * PER) * 8);
    }
    cluster_arrive_relaxed();   // waited for before the first push, after GEMM 1: no peer pushes into an uninitialised barrier
  }

  // ---- data half: sampler + image rows 6c .. 6c+9 (280 contiguous pixels per sample), before the PDL wait ----------------
  const int call = a.calls != nullptr ? a.calls[l] : 0;
  const BatchGeom bg = batch_geom<true>(a, l, call);
  if (tid < MS) {
    int idx = 0, lab = 0; float ok = 0.f;
    const uint32_t t = (uint32_t)(bsplit * MS + tid);
    if (t < bg.bs) {
      ok = 1.f;
      idx = a.direct ? (int)(l * a.batch + t) : bg.shard_off + (int)feistel_permute(bg.start + t, bg.m, bg.key);
      lab = (int)a.y[idx];
    }
    sm.sidx[tid] = idx; sm.valid[tid] = ok; sm.label[tid] = lab;
  }
  if constexpr (!kDoublePix)
    if (tid < 256) sm.lut[tid] = ((double)tid * (1.0 / 255.0) - pmean) * pis;
  __syncthreads();
  // u8 rows: 35 8-byte chunks per sample (the window starts at byte 168 c, 8-byte aligned); fp32 rows: 70 float4
  constexpr int NU8 = (MS * 35 + NT - 1) / NT, NF4 = kDoublePix ? (MS * 70 + NT - 1) / NT : 1;
  uint2 pu[NU8]; float4 pf[NF4];
  if (u8) {
#pragma unroll
    for (int i = 0; i < NU8; ++i) {
      const int o = tid + i * NT;
      pu[i] = make_uint2(0, 0);
      if (o < MS * 35) {
        const int s = o / 35, q = o - s * 35;
        if (sm.valid[s] != 0.f)
          pu[i] = *reinterpret_cast<const uint2*>(reinterpret_cast<const unsigned char*>(a.x) + (size_t)sm.sidx[s] * 784 + 6 * HW * c + 8 * q);
      }
    }
  } else if constexpr (kDoublePix) {
#pragma unroll
    for (int i = 0; i < NF4; ++i) {
      const int o = tid + i * NT;
      pf[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (o < MS * 70) {
        const int s = o / 70, q = o - s * 70;
        if (sm.valid[s] != 0.f)
          pf[i] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.x) + (size_t)sm.sidx[s] * 784 + 6 * HW * c + 4 * q);
      }
    }
  }
  // the rows are data, not parameters: they are normalised into shared memory before the PDL wait
  if (u8) {
#pragma unroll
    for (int i = 0; i < NU8; ++i) {
      const int o = tid + i * NT;
      if (o < MS * 35) {
        const int s = o / 35, q = o - s * 35;
        if constexpr (kDoublePix) {
          const uint32_t w[2] = {pu[i].x, pu[i].y};
          double* dst = imgd + s * PXS + 8 * q;
#pragma unroll
          for (int j = 0; j < 8; ++j) dst[j] = ((double)((w[j >> 2] >> (8 * (j & 3))) & 0xff) * (1.0 / 255.0) - pmean) * pis;
        } else {
          *reinterpret_cast<uint2*>(sm.img + s * PXR + 8 * q) = pu[i];
        }
      }
    }
  } else if constexpr (kDoublePix) {
#pragma unroll
    for (int i = 0; i < NF4; ++i) {
      const int o = tid + i * NT;
      if (o < MS * 70) {
        double* dst = imgd + (o / 70) * PXS + 4 * (o % 70);
        dst[0] = pf[i].x; dst[1] = pf[i].y; dst[2] = pf[i].z; dst[3] = pf[i].w;
      }
    }
  }
  stamp(prof, 1, tid);
  pdl_wait();                 // the parameters of this step are final
  pdl_launch_dependents();
  stamp(prof, 2, tid);

  // ---- W1 slice [64 j][108 k] (three 36-double runs per row, 16-byte chunks), b1, b2: asynchronous copies that land
  //      while the conv runs.  The 78 conv weights and biases and w2 (re-laid out, so not a plain copy) are loaded
  //      through registers, their L2 round trip under the copy issue; only these are waited for before the conv ------------
  constexpr int NW2 = (NCLS * HID + NT - 1) / NT;
  double wcv = 0.0, w2v[NW2];
  if (tid < 75) wcv = __ldcg(th + a.off_wc + tid);
  else if (tid < 78) wcv = __ldcg(th + a.off_bc + (tid - 75));
#pragma unroll
  for (int i = 0; i < NW2; ++i) {
    const int o = tid + i * NT;
    w2v[i] = o < NCLS * HID ? __ldcg(th + a.off_w2 + o) : 0.0;
  }
  for (int o = tid; o < HID * KC / 2; o += NT) {
    const int j = o / (KC / 2), r = o - j * (KC / 2), ch = r / (CELLS / 2), q = 2 * (r - ch * (CELLS / 2));
    cp_async16(sm.w + j * WS + ch * CELLS + q, th + a.off_w1 + (size_t)j * FC1_IN + ch * NPOOL + CELLS * c + q);
  }
  if (tid < HID / 2) cp_async16(sm.b1 + 2 * tid, th + a.off_b1 + 2 * tid);
  else if (tid >= 32 && tid < 32 + NCLS / 2) cp_async16(sm.b2 + 2 * (tid - 32), th + a.off_b2 + 2 * (tid - 32));
  cp_async_commit();
  if (tid < 78) sm.wc[tid] = wcv;
#pragma unroll
  for (int i = 0; i < NW2; ++i) {
    const int o = tid + i * NT;
    if (o < NCLS * HID) sm.w2[(o / HID) * HR + hr(o % HID)] = w2v[i];
  }
  __syncthreads();
  stamp(prof, 3, tid);

  // ---- conv + ReLU + maxpool: one (sample, pooled cell) per item.  Two rows of the 6x6 patch are in fp64 registers at a
  //      time, one new row per tap row, and the four pool positions of all three channels accumulate together; each
  //      accumulator takes its products in (ky, kx) order ------------------------------------------------------------------
  for (int it = tid; it < MS * CELLS; it += NT) {
    const int s = it / CELLS, cell = it - s * CELLS;
    const int pr = cell / PHW, px = cell - pr * PHW;
    const int p0 = (2 * pr) * HW + 2 * px;
    auto patch_row = [&](double (&x)[6], int r) {
      if constexpr (kDoublePix) {
        // a patch row is six consecutive doubles starting at an even column: three 16-byte loads
        const double* src = imgd + s * PXS + p0 + r * HW;
#pragma unroll
        for (int q = 0; q < 6; q += 2) {
          const double2 v = *reinterpret_cast<const double2*>(src + q);
          x[q] = v.x; x[q + 1] = v.y;
        }
      } else {
#pragma unroll
        for (int q = 0; q < 6; ++q) x[q] = pix(s, p0 + r * HW + q);
      }
    };
    double acc[F][4], x0[6], x1[6];
#pragma unroll
    for (int ch = 0; ch < F; ++ch)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[ch][i] = 0;
    patch_row(x0, 0);
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
      patch_row(x1, ky + 1);
#pragma unroll
      for (int kx = 0; kx < KS; ++kx)
#pragma unroll
        for (int ch = 0; ch < F; ++ch) {
          const double w = sm.wc[ch * 25 + ky * 5 + kx];
          acc[ch][0] += w * x0[kx]; acc[ch][1] += w * x0[kx + 1];
          acc[ch][2] += w * x1[kx]; acc[ch][3] += w * x1[kx + 1];
        }
#pragma unroll
      for (int q = 0; q < 6; ++q) x0[q] = x1[q];
    }
    const bool ok = sm.valid[s] != 0.f;
#pragma unroll
    for (int ch = 0; ch < F; ++ch) {
      const double a00 = acc[ch][0], a01 = acc[ch][1], a10 = acc[ch][2], a11 = acc[ch][3];
      double m = a00; int ai = 0;                      // first maximum wins, like ATen's max_pool2d
      if (a01 > m) { m = a01; ai = 1; }
      if (a10 > m) { m = a10; ai = 2; }
      if (a11 > m) { m = a11; ai = 3; }
      m += sm.wc[75 + ch];
      m = (ok && m > 0.0) ? m : 0.0;
      sm.a[s * WS + ch * CELLS + cell] = m;
      sm.arg[s * KC + ch * CELLS + cell] = (unsigned char)(ai | (m > 0.0 ? 4 : 0));
    }
  }
  cp_async_wait<0>();   // this thread's W1 / w2 / b1 / b2 chunks have landed; the barrier publishes everyone's
  __syncthreads();
  stamp(prof, 4, tid);

  // ---- GEMM 1 (DMMA): partial H_c[s][j] = sum_k A[s][k] W[j][k] over this CTA's 108 inputs.  MS / 16 x 8 tiles of 16 x 8,
  //      NJ1 adjacent column tiles per warp (16 of the 20 warps busy at MS >= 32), the whole K range per tile: no split-K.
  //      kPush: accumulator pairs go straight to the owner of each sample (s / NO), invalid samples' zero rows included,
  //      so every byte count is static -----------------------------------------------------------------------------------
  {
    constexpr int NJ1 = MS == 64 ? 2 : 1, NGRP = 8 / NJ1;
    const bool busy = warp < (MS / 16) * NGRP;
    const int m0 = 16 * (warp / NGRP), n0 = 8 * NJ1 * (warp % NGRP);
    double acc[NJ1][4];
    zero(acc);
    if (busy) gemm_k<NJ1, KC>(acc, m0, n0, lane, at(sm.a, WS), at_t(sm.w, WS));
    if constexpr (kPush) {
      cluster_wait();
      if (busy) {
#pragma unroll
        for (int j = 0; j < NJ1; ++j)
#pragma unroll
          for (int i = 0; i < 4; i += 2) {
            const int s = frow(m0, lane, i), r = s / NO;
            st_async(map_to(sm.hin + (c * NO + s - r * NO) * HID + fcol(n0 + 8 * j, lane, i), (uint32_t)r), acc[j][i],
                     acc[j][i + 1], map_to(&sm.bar[0], (uint32_t)r));
          }
      }
    } else if (busy) {
#pragma unroll
      for (int j = 0; j < NJ1; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) sm.h[frow(m0, lane, i) * HS + fcol(n0 + 8 * j, lane, i)] = acc[j][i];
    }
  }
  stamp(prof, 5, tid);
  if constexpr (kPush) {
    if (warp < NO) mbarrier_wait_parity_cluster(&sm.bar[0], 0);   // the four partial H of this CTA's samples
  } else {
    cluster_sync();                                      // #1: all four partial H are in shared memory
  }
  stamp(prof, 6, tid);
  // every CTA of the cluster has read `call`: it had before its partial H, which thread 0 has received (kPush) or which
  // barrier #1 published
  if (c == 0 && tid == 0 && a.calls != nullptr) {
    if (a.arrive == nullptr || nsplit == 1) a.calls[l] = call + 1;
    else if (atomicAdd(a.arrive + l, 1u) == (unsigned)nsplit - 1) { a.arrive[l] = 0; a.calls[l] = call + 1; }
  }

  // ---- reduce-scatter of H + fc2 / loss / their backward for this CTA's samples s0 .. s0 + NO - 1: one warp per sample,
  //      lanes own hidden units j = lane and lane + 32; from the DSMEM sum to dh the warp needs no block barrier --------
  const int s0 = c * NO;
  const double inv_bs = 1.0 / (double)(bg.bs ? bg.bs : 1);
  if (warp < NO) {
    const int sl = warp, s = s0 + sl;
    double hv[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int j = lane + 32 * q;
      const double* src = sm.h + s * HS + j;
      double v = sm.b1[j];
#pragma unroll
      for (int r = 0; r < CL; ++r) {
        if constexpr (kPush) v += sm.hin[(r * NO + sl) * HID + j];
        else v += ld_dsmem(map_to(src, (uint32_t)r));
      }
      hv[q] = v > 0.0 ? v : 0.0;
      sm.h_loc[sl * HR + hr(j)] = hv[q];
    }
    __syncwarp();
    // logits: 4 lanes per class, each summing 16 consecutive hidden units, folded over lane bits 0 and 1; 40 partial sums,
    // so lanes 0 .. 7 take a second one (classes 8 and 9)
    double zp[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int o = lane + 32 * r, cc = o >> 2, part = o & 3;
      double v = 0.0;
      if (o < 4 * NCLS) {
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) v += sm.h_loc[sl * HR + part * 17 + jj] * sm.w2[cc * HR + part * 17 + jj];
      }
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      zp[r] = v;
    }
    static_assert(NCLS > 8 && NCLS <= 16, "two rounds of four lanes per class");
    const double z0 = __shfl_sync(0xffffffffu, zp[0], (4 * lane) & 31), z1 = __shfl_sync(0xffffffffu, zp[1], (4 * lane) & 31);
    // log-softmax + NLL, one lane per class
    const bool cls = lane < NCLS;
    const double zc = cls ? (lane < 8 ? z0 : z1) + sm.b2[lane] : -1.0e300;
    const double mx = wmax(zc);
    const double se = warp_sum(cls ? exp(zc - mx) : 0.0);
    const double lse = mx + log(se);
    const int y = sm.label[s];
    const double ok = (double)sm.valid[s];
    const double dzc = cls ? ok * inv_bs * (exp(zc - lse) - (lane == y ? 1.0 : 0.0)) : 0.0;
    if (cls) sm.dz[sl * 16 + lane] = dzc;
    if (lane == y) sm.red[sl] = ok * (lse - zc);
    // dh = dz . W2, masked by ReLU'(h)
    double dh[2] = {0.0, 0.0};
#pragma unroll
    for (int cc = 0; cc < NCLS; ++cc) {
      const double d = __shfl_sync(0xffffffffu, dzc, cc);
      dh[0] += d * sm.w2[cc * HR + hr(lane)];
      dh[1] += d * sm.w2[cc * HR + hr(lane + 32)];
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      dh[q] = hv[q] > 0.0 ? dh[q] : 0.0;
      sm.dh_loc[sl * HID + lane + 32 * q] = dh[q];
    }
    if constexpr (kPush) {
      // lane i pushes hidden units 2i, 2i + 1 of sample s into the dH tile of every CTA, this one included
      const int e = (2 * lane) & 31;
      const double e0 = __shfl_sync(0xffffffffu, dh[0], e), e1 = __shfl_sync(0xffffffffu, dh[1], e);
      const double o0 = __shfl_sync(0xffffffffu, dh[0], e + 1), o1 = __shfl_sync(0xffffffffu, dh[1], e + 1);
#pragma unroll
      for (int r = 0; r < CL; ++r)
        st_async(map_to(sm.h + s * HS + 2 * lane, (uint32_t)r), lane < 16 ? e0 : e1, lane < 16 ? o0 : o1,
                 map_to(&sm.bar[1], (uint32_t)r));
    }
  }
  __syncthreads();
  // the fc2 / b1 / b2 / loss shares: kPush sends entry o straight to the CTA that reduces it; otherwise the peers read it
  auto share = [&](int o, double v) {
    if constexpr (kPush) {
      const int e = o - PART_B1, q = e / PER;
      st_async(map_to(sm.shr + c * PER + (e - q * PER), (uint32_t)q), v, map_to(&sm.bar[2], (uint32_t)q));
    } else {
      sm.part[o] = v;
    }
  };
  for (int o = tid; o < NCLS * HID; o += NT) {
    const int cc = o >> 6, j = o & 63;
    double v = 0.0;
    for (int sl = 0; sl < NO; ++sl) v += sm.dz[sl * 16 + cc] * sm.h_loc[sl * HR + hr(j)];
    share(PART_W2 + o, v);
  }
  if (tid < HID) {
    double v = 0.0;
    for (int sl = 0; sl < NO; ++sl) v += sm.dh_loc[sl * HID + tid];
    share(PART_B1 + tid, v);
  } else if (tid >= 64 && tid < 64 + NCLS) {
    double v = 0.0;
    for (int sl = 0; sl < NO; ++sl) v += sm.dz[sl * 16 + (tid - 64)];
    share(PART_B2 + (tid - 64), v);
  } else if (tid == 96) {
    double v = 0.0;
    for (int sl = 0; sl < NO; ++sl) v += sm.red[sl];
    share(PART_LOSS, v * inv_bs);
  }
  stamp(prof, 7, tid);
  if constexpr (kPush) mbarrier_wait_parity_cluster(&sm.bar[1], 0);   // all MS dH rows
  else cluster_sync();                                   // #2: every owner's dH rows and fc2 / b1 / loss shares are final
  stamp(prof, 8, tid);
  // this split's gradient row, formed where it is written: a pointer held from here to the end would cost two registers
  // through GEMM 2 and the conv grads, and the kernel has 96 per thread
  auto grad_row = [&]() { return reinterpret_cast<double*>(a.grad_part) + ((size_t)l * nsplit + bsplit) * a.n_pad; };
  // CTA c reduces entries PART_B1 + c PER + i of the fc2 / b1 / b2 / loss shares over the cluster, ranks in order
  auto reduce_share = [&](int i) {
    const int o = PART_B1 + c * PER + i;
    if (o >= PART_N) return;
    double* gp = grad_row();
    double v = 0.0;
#pragma unroll
    for (int r = 0; r < CL; ++r) {
      if constexpr (kPush) v += sm.shr[r * PER + i];
      else v += ld_dsmem(map_to(sm.part + o, (uint32_t)r));
    }
    if (o < PART_W2) gp[a.off_b1 + (o - PART_B1)] = v;
    else if (o < PART_B2) gp[a.off_w2 + (o - PART_W2)] = v;
    else if (o < PART_LOSS) gp[a.off_b2 + (o - PART_B2)] = v;
    else {
      a.loss_part[l * nsplit + bsplit] = (float)v;
      if (a.loss_mirror != nullptr) a.loss_mirror[l * nsplit + bsplit] = (float)v;
    }
  };
  if constexpr (!kPush) {
    // (the peers stay resident until the last barrier)
    if (tid < PER) reduce_share(tid);
    // ---- gather all MS dH rows from their owners into the partial-H tile (every peer finished reading it before #2) ---------
    for (int o = tid; o < MS * HID; o += NT) {
      const int s = o >> 6, j = o & 63, r = s / NO;
      sm.h[s * HS + j] = ld_dsmem(map_to(sm.dh_loc + (s - r * NO) * HID + j, (uint32_t)r));
    }
    __syncthreads();
  }
  stamp(prof, 9, tid);

  // ---- GEMM 2 (DMMA): da1_c[s][k] = sum_j dH[s][j] W[j][k], MS / 16 x KT / 2 pairs of adjacent 16 x 8 tiles, accumulators
  //      held in registers until every warp is done reading W; then da1 [k][s] (sample-minor for the conv-grad pass, masked
  //      by ReLU'(a1)) is written over the dead W slice.  A stays intact for GEMM 3 --------------------------------------------
  constexpr int NP2 = (MS / 16) * (KT / 2), NR2 = (NP2 + NT / 32 - 1) / (NT / 32);
  static_assert(KT % 2 == 0 && KC * MS + (NT / 32) * 16 <= HID * WS, "da1 and the conv-grad warp sums fit in the W slice");
  double acc2[NR2][2][4];
#pragma unroll
  for (int r = 0; r < NR2; ++r) {
    zero(acc2[r]);
    const int p = warp + r * (NT / 32);
    if (p < NP2) gemm_k<2, HID>(acc2[r], 16 * (p / (KT / 2)), 16 * (p % (KT / 2)), lane, at(sm.h, HS), at(sm.w, WS));
  }
  __syncthreads();      // every read of W is done
  stamp(prof, 10, tid);
  double* da1 = sm.w;
#pragma unroll
  for (int r = 0; r < NR2; ++r) {
    const int p = warp + r * (NT / 32);
    if (p < NP2) {
      const int m0 = 16 * (p / (KT / 2)), n0 = 16 * (p % (KT / 2));
#pragma unroll
      for (int jt = 0; jt < 2; ++jt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int s = frow(m0, lane, i), k = fcol(n0 + 8 * jt, lane, i);
          if (k < KC) da1[k * MS + s] = (sm.arg[s * KC + k] & 4) ? acc2[r][jt][i] : 0.0;
        }
    }
  }
  __syncthreads();
  stamp(prof, 11, tid);
  // ---- GEMM 3 (DMMA) on warps 16 .. 19, one per SM sub-partition: dW1_c[j][k] = sum_s dH[s][j] A[s][k].  Warp 16 + q owns
  //      hidden rows 16q .. 16q+15 and all KT column tiles, two at a time: two independent DMMA chains share the dH
  //      fragments (seven, with their next fragments in flight, do not fit in 96 registers).  Tiles go straight to the
  //      gradient row (column pairs as 16-byte stores).  Meanwhile warps 0 .. 14 run their conv-grad rows and warp 15 the
  //      bias sums, so the FP64 pipe of every sub-partition is busy while its tensor cores run GEMM 3.  No barrier on
  //      either side -----------------------------------------------------------------------------------------------------
  constexpr int W3 = NT / 32 - HID / 16, NJ3 = 2;   // first GEMM 3 warp; column tiles per pass
  static_assert(KT % NJ3 == 0, "GEMM 3 passes cover the column tiles");
  if (warp >= W3) {
    // kPush: the shares of this CTA's quarter arrived while GEMM 2 ran; these warps reduce them first, as they end about
    // 3 us before the conv-gradient warps
    if constexpr (kPush) {
      mbarrier_wait_parity_cluster(&sm.bar[2], 0);
      for (int i = tid - W3 * 32; i < PER; i += NT - W3 * 32) reduce_share(i);
    }
    double* gp = grad_row();
    const int m0 = 16 * (warp - W3);
#pragma unroll 1
    for (int n0 = 0; n0 < 8 * KT; n0 += 8 * NJ3) {
      double acc[NJ3][4];
      zero(acc);
      gemm_k<NJ3, MS>(acc, m0, n0, lane, at_t(sm.h, HS), at(sm.a, WS));
#pragma unroll
      for (int jt = 0; jt < NJ3; ++jt)
#pragma unroll
        for (int i = 0; i < 4; i += 2) {
          const int j = frow(m0, lane, i), k = fcol(n0 + 8 * jt, lane, i);   // k even: k and k + 1 share a channel run
          if (k < KC) {
            // __stcg keeps the pair one 16-byte store: a plain double2 assignment was split into two 8-byte stores,
            // which doubled the partial-sector writes of the 55 KB dW1 slice
            const int ch = k / CELLS, cell = k - ch * CELLS;
            __stcg(reinterpret_cast<double2*>(gp + a.off_w1 + (size_t)j * FC1_IN + ch * NPOOL + CELLS * c + cell),
                   make_double2(acc[jt][i], acc[jt][i + 1]));
          }
        }
    }
    stamp(prof, 12, tid - W3 * 32);      // lane 0 of warp W3: its GEMM 3 stores are issued
  }
  // ---- conv grads without gathers: warps 3ky .. 3ky+2 own tap row ky of all three channels.  A thread walks whole pooled
  //      rows (sample s, pooled row pr, px = 0 .. 11) with columns 2px .. 2px+5 of patch rows 2pr+ky and 2pr+ky+1 in
  //      registers, two new columns per cell.  Each cell's gradient goes to all four pool positions, zero except at its
  //      argmax, so every lane runs the same 20 DFMA per channel and no address depends on the argmax.  Warp 15 sums the
  //      bias gradients.  Every warp folds its sums over its lanes and a tap row's three warp sums are added in warp order ---
  constexpr int KW = 3, NRUN = MS * 3;   // warps per tap row; (sample, pooled row) runs
  static_assert(KS * KW < NT / 32 && F * KS <= 16, "conv-grad work split");
  double* wsums = sm.w + KC * MS;        // [NT / 32][16], behind da1
  // columns p, p + 1 (p even) of sample s's rows: one 16-byte load from the double rows
  auto pix2 = [&](int s, int p) -> double2 {
    if constexpr (kDoublePix) return *reinterpret_cast<const double2*>(imgd + s * PXS + p);
    else return make_double2(pix(s, p), pix(s, p + 1));
  };
  if (warp < KS * KW) {
    const int ky = warp / KW;
    double acc[16];                      // [ch][kx]; slot 15 stays zero
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.0;
#pragma unroll 1
    for (int r = tid - ky * KW * 32; r < NRUN; r += KW * 32) {
      const int s = r % MS, pr = r / MS;                   // consecutive lanes take consecutive samples
      const int rb = (2 * pr + ky) * HW;
      double x0[6], x1[6];
#pragma unroll
      for (int px = 0; px < PHW; ++px) {
        const int p = rb + 2 * px;
        if (px == 0) {
#pragma unroll
          for (int q = 0; q < 6; q += 2) {
            const double2 u = pix2(s, p + q), v = pix2(s, p + HW + q);
            x0[q] = u.x; x0[q + 1] = u.y; x1[q] = v.x; x1[q + 1] = v.y;
          }
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) { x0[q] = x0[q + 2]; x1[q] = x1[q + 2]; }
          const double2 u = pix2(s, p + 4), v = pix2(s, p + HW + 4);
          x0[4] = u.x; x0[5] = u.y; x1[4] = v.x; x1[5] = v.y;
        }
#pragma unroll
        for (int ch = 0; ch < F; ++ch) {
          const int k = ch * CELLS + pr * PHW + px;
          const double g = da1[k * MS + s];
          const int ai = sm.arg[s * KC + k] & 3;
          const double g00 = ai == 0 ? g : 0.0, g01 = ai == 1 ? g : 0.0, g10 = ai == 2 ? g : 0.0, g11 = ai == 3 ? g : 0.0;
#pragma unroll
          for (int kx = 0; kx < KS; ++kx) {
            double& t = acc[ch * KS + kx];
            t = fma(g00, x0[kx], t); t = fma(g01, x0[kx + 1], t);
            t = fma(g10, x1[kx], t); t = fma(g11, x1[kx + 1], t);
          }
        }
      }
    }
    warp_reduce_scatter16(acc, lane);
    if ((lane & 1) == 0 && (lane >> 1) < F * KS) wsums[warp * 16 + (lane >> 1)] = acc[0];
  } else if (warp == KS * KW) {
#pragma unroll 1
    for (int ch = 0; ch < F; ++ch) {
      double v = 0.0;
      for (int o = lane; o < CELLS * MS; o += 32) v += da1[ch * CELLS * MS + o];
      v = warp_sum(v);
      if (lane == 0) wsums[warp * 16 + ch] = v;
    }
  }
  __syncthreads();
  // this CTA's share goes straight into rank 0's collection buffer.  kPush: rank 0's partial-H buffer, last read by its head
  // warps before they pushed dH, which every peer has received before it gets here.  Otherwise its h_loc rows, dead since
  // barrier #2
  double* cin = kPush ? sm.hin : sm.h_loc;
  if (tid < 78) {
    double v = 0.0;
    if (tid < 75) {
      const int ch = tid / 25, t = tid - ch * 25, ky = t / KS, kx = t - ky * KS;
#pragma unroll
      for (int w = 0; w < KW; ++w) v += wsums[(ky * KW + w) * 16 + ch * KS + kx];
    } else {
      v = wsums[KS * KW * 16 + (tid - 75)];
    }
    st_dsmem(map_to(cin + c * 80 + tid, 0u), v);
  }
  stamp(prof, 13, tid);
  cluster_sync();                                        // #3: all four conv-gradient shares are in rank 0's buffer
  if (c == 0 && tid < 78) {
    double* gp = grad_row();
    double v = 0.0;
#pragma unroll
    for (int r = 0; r < CL; ++r) v += cin[r * 80 + tid];
    gp[tid < 75 ? a.off_wc + tid : a.off_bc + (tid - 75)] = v;
  }
  stamp(prof, 14, tid);
}

template <int MS>
static cudaError_t prepare_ms() {
  static cudaError_t prep = cudaFuncSetAttribute(mnist_cl64_train_kernel<MS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<MS>));
  return prep;
}

template <int MS>
static cudaError_t launch_ms(const Args& a, const GenericShape& gs, cudaStream_t st) {
  const cudaError_t prep = prepare_ms<MS>();
  if (prep != cudaSuccess) return prep;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(CL, 64 / MS, a.L); cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = sizeof(Smem<MS>); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  static const bool no_pdl = getenv("NNDT_NO_PDL") != nullptr;
  cfg.attrs = attr; cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, mnist_cl64_train_kernel<MS>, a, gs);
}

template <int MS>
static int max_clusters_ms() {
  if (prepare_ms<MS>() != cudaSuccess) { cudaGetLastError(); return 0; }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(CL, 1, 1); cfg.blockDim = dim3(NT); cfg.dynamicSmemBytes = sizeof(Smem<MS>);
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, mnist_cl64_train_kernel<MS>, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

}  // namespace cl64

cudaError_t launch_train_cl64(const Args& a, const GenericShape& gs, int nsplit, cudaStream_t st) {
  switch (nsplit) {
    case 1: return cl64::launch_ms<64>(a, gs, st);
    case 2: return cl64::launch_ms<32>(a, gs, st);
    case 4: return cl64::launch_ms<16>(a, gs, st);
  }
  return cudaErrorInvalidValue;
}

int cl64_max_active_clusters(int nsplit) {
  switch (nsplit) {
    case 1: return cl64::max_clusters_ms<64>();
    case 2: return cl64::max_clusters_ms<32>();
    case 4: return cl64::max_clusters_ms<16>();
  }
  return 0;
}

int cl64_cluster_ctas() { return cl64::CL; }

}  // namespace mnist
}  // namespace nndt
