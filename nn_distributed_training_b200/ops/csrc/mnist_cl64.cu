// float64 training kernel of the paper's MNISTConvNet(3, 5, 64) at batch <= 64: the K-split thread-block-cluster
// decomposition of mnist_tc.cu with the contractions on the fp64 CUDA cores (fp64 operands would need the DMMA
// tensor-core path and its fragment layouts for the same K-split; the vector DFMA units carry it here).  This is the kernel behind the framework's float64 arm — the
// precision the reference runs end to end (experiments/dist_mnist_ex.py:19) — and replaces the batch-split generic
// kernel (mnist_generic.cu) there, which streams the 221 KB fp64 W1 matrix three times per CTA.
//
// A node is `nsplit` clusters of 6 CTAs (MS = 64 / nsplit samples each); CTA c owns pooled rows {2c, 2c+1} of all three
// channels = 72 of the 432 fc1 inputs for all MS samples: conv+ReLU+pool -> A_c [MS x 72]; H_c = A_c . W1_c^T reduced
// over the cluster through distributed shared memory (reduce-scatter by samples, fc2 / loss / backward on the owners, dH
// rows gathered back); da1_c = dH . W1_c and dW1_c = dH^T . A_c are local; dW1_c goes straight to its columns of the
// gradient row; small gradients are reduced by rank 0 through DSMEM.  One gradient partial row per cluster.
// GEMM tiling: a thread owns 2 rows x 4-5 strided columns; with rows padded to 73 / 65 doubles every operand read is
// either a broadcast or conflict free, so the loops run at the DFMA rate.
#include <type_traits>

#include "mnist_device.cuh"

namespace nndt {
namespace mnist {

namespace cl64 {

constexpr int NT = 512, CL = 6, CELLS = 24, KC = 72, WS = 73, HS = 65;
constexpr int PART_WC = 0, PART_BC = 75, PART_B1 = 78, PART_W2 = 142, PART_B2 = 782, PART_LOSS = 792, PART_N = 793;

struct Smem {
  double w[64 * WS];         // W1 slice [j][k], k = ch * 24 + cell; later da1 [s][72]
  double a[64 * WS];         // A tile [s][k]; later (with dh) the scratch of the conv-grad reduction
  double dh[64 * HS];        // dH [s][j]; before that, split-K partial sums of GEMM 1
  double hpart[64 * HS];     // partial H [s][j] (read by the peers); later split-K partial sums of GEMM 2
  alignas(16) unsigned char img[64 * 224 * 4];   // image rows 4c .. 4c+7: MS <= 32: normalised doubles [MS][224]; MS = 64: raw floats
  double h_loc[11 * 64];     // later (rank 0) the six CTAs' conv-gradient shares [6][80]
  double dh_loc[11 * 64];
  double part[800];
  double w2[NCLS * HID];
  double b1[HID];
  double b2[16];
  double wc[80];
  double z[11 * 16];
  double dz[11 * 16];
  double red[16];
  int sidx[64];
  int label[64];
  float valid[64];
  unsigned char arg[64 * KC];
};
static_assert(sizeof(Smem) <= 227 * 1024, "shared memory budget");
static_assert(6 * 80 <= 11 * 64, "conv shares fit h_loc");

NNDT_DEVINL double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
NNDT_DEVINL double wmax(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
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
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int l = blockIdx.z, bsplit = blockIdx.y, nsplit = gridDim.y;
  const int c = (int)cluster_rank();
  const double* th = reinterpret_cast<const double*>(a.theta) + (size_t)l * a.n_pad;
  auto own_lo = [](int r) { return (MS * r + CL - 1) / CL; };
  const double pmean = gs.mean, pis = gs.inv_std;
  const bool u8 = a.x_is_u8 != 0;
  // pixels: with MS <= 32 samples the 8 x 28 slabs fit as normalised doubles, so conv and conv-grad read fp64 directly
  constexpr bool kDoublePix = MS <= 32;
  using PT = typename std::conditional<kDoublePix, double, float>::type;
  PT* img = reinterpret_cast<PT*>(sm.img);
  auto pix = [&](PT v) -> double {
    if constexpr (kDoublePix) return v;
    else return u8 ? ((double)v * (1.0 / 255.0) - pmean) * pis : (double)v;
  };
  long long* prof = a.prof != nullptr ? a.prof + ((l * nsplit + bsplit) * CL + c) * 64 : nullptr;
  stamp(prof, 0, tid);

  // ---- data half: sampler + image rows 4c .. 4c+7 (224 contiguous pixels per sample), before the PDL wait ---------------
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
  __syncthreads();
  constexpr int NU8 = (MS * 14 + NT - 1) / NT, NF4 = (MS * 56 + NT - 1) / NT;
  uint4 pu[NU8]; float4 pf[NF4];
  if (u8) {
#pragma unroll
    for (int i = 0; i < NU8; ++i) {
      const int o = tid + i * NT;
      pu[i] = make_uint4(0, 0, 0, 0);
      if (o < MS * 14) {
        const int s = o / 14, q = o - s * 14;
        if (sm.valid[s] != 0.f)
          pu[i] = *reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(a.x) + (size_t)sm.sidx[s] * 784 + 112 * c + 16 * q);
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < NF4; ++i) {
      const int o = tid + i * NT;
      pf[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (o < MS * 56) {
        const int s = o / 56, q = o - s * 56;
        if (sm.valid[s] != 0.f)
          pf[i] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.x) + (size_t)sm.sidx[s] * 784 + 112 * c + 4 * q);
      }
    }
  }
  stamp(prof, 1, tid);
  pdl_wait();                 // the parameters of this step are final
  pdl_launch_dependents();
  stamp(prof, 2, tid);

  // ---- W1 slice [64 j][72 k] (three 24-column runs per row): loads in flight while the pixels are converted --------------
  constexpr int NW = (HID * KC + NT - 1) / NT;
  double wreg[NW];
#pragma unroll
  for (int i = 0; i < NW; ++i) {
    const int o = tid + i * NT;
    wreg[i] = 0.0;
    if (o < HID * KC) {
      const int j = o / KC, r = o - j * KC, ch = r / CELLS, cell = r - ch * CELLS;
      wreg[i] = __ldcg(th + a.off_w1 + (size_t)j * FC1_IN + ch * NPOOL + CELLS * c + cell);
    }
  }
  for (int o = tid; o < NCLS * HID; o += NT) sm.w2[o] = __ldcg(th + a.off_w2 + o);
  if (tid < 75) sm.wc[tid] = __ldcg(th + a.off_wc + tid);
  else if (tid < 78) sm.wc[tid] = __ldcg(th + a.off_bc + (tid - 75));
  else if (tid >= 96 && tid < 96 + HID) sm.b1[tid - 96] = __ldcg(th + a.off_b1 + (tid - 96));
  else if (tid >= 160 && tid < 160 + NCLS) sm.b2[tid - 160] = __ldcg(th + a.off_b2 + (tid - 160));
  if (u8) {
#pragma unroll
    for (int i = 0; i < NU8; ++i) {
      const int o = tid + i * NT;
      if (o < MS * 14) {
        const int s = o / 14, q = o - s * 14;
        const uint32_t w[4] = {pu[i].x, pu[i].y, pu[i].z, pu[i].w};
        PT* dst = img + s * 224 + 16 * q;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const double v = (double)((w[j >> 2] >> (8 * (j & 3))) & 0xff);
          if constexpr (kDoublePix) dst[j] = (v * (1.0 / 255.0) - pmean) * pis; else dst[j] = (float)v;
        }
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < NF4; ++i) {
      const int o = tid + i * NT;
      if (o < MS * 56) {
        PT* dst = img + (o / 56) * 224 + 4 * (o % 56);
        dst[0] = (PT)pf[i].x; dst[1] = (PT)pf[i].y; dst[2] = (PT)pf[i].z; dst[3] = (PT)pf[i].w;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NW; ++i) {
    const int o = tid + i * NT;
    if (o < HID * KC) sm.w[(o / KC) * WS + (o % KC)] = wreg[i];
  }
  __syncthreads();
  stamp(prof, 3, tid);

  // ---- conv + ReLU + maxpool: one (sample, pooled cell) per item, the 6x6 patch in fp64 registers ---------------------------
  for (int it = tid; it < MS * CELLS; it += NT) {
    const int s = it / CELLS, cell = it - s * CELLS;
    const int pr = cell / PHW, px = cell - pr * PHW;
    const PT* src = img + s * 224 + (2 * pr) * HW + 2 * px;
    double patch[6][6];
    if constexpr (kDoublePix) {
      // a patch row is six consecutive doubles starting at the even column 2 px: three 16-byte loads, and consecutive lanes
      // (consecutive px) read consecutive 16-byte chunks -> half the shared-memory wavefronts of 8-byte loads at stride 2
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int q = 0; q < 6; q += 2) {
          const double2 v = *reinterpret_cast<const double2*>(src + r * HW + q);
          patch[r][q] = v.x; patch[r][q + 1] = v.y;
        }
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int q = 0; q < 6; ++q) patch[r][q] = pix(src[r * HW + q]);
    }
    const bool ok = sm.valid[s] != 0.f;
#pragma unroll 1
    for (int ch = 0; ch < F; ++ch) {
      double a00 = 0, a01 = 0, a10 = 0, a11 = 0;
#pragma unroll
      for (int ky = 0; ky < KS; ++ky)
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const double w = sm.wc[ch * 25 + ky * 5 + kx];
          a00 += w * patch[ky][kx]; a01 += w * patch[ky][kx + 1];
          a10 += w * patch[ky + 1][kx]; a11 += w * patch[ky + 1][kx + 1];
        }
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
  __syncthreads();
  stamp(prof, 4, tid);

  // ---- GEMM 1: H_c[s][j] = sum_k A[s][k] W[j][k].  Register tile 4 rows x 4 columns (rows tr + RQ i, columns tc + 16 i):
  //      per k a warp issues 4 + 4 shared-memory wavefronts for 16 DFMA instructions.  Split-K over NG = 512 / (4 MS) thread
  //      groups; group g writes its partial tile to P_g (the contiguous dh + hpart arrays hold NG x MS = 128 rows) and the
  //      partials are summed in fixed order (deterministic) into the rows the peers read.
  constexpr int RQ = MS / 4, GT = MS * 4, NG = NT / GT, KG = KC / NG;
  static_assert(KC % NG == 0 && NG * MS == 128, "split-K geometry");
  const int grp = tid / GT, tg = tid - grp * GT, tr = tg >> 4, tc = tg & 15;
  {
    double acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[r][i] = 0.0;
#pragma unroll 2
    for (int k = grp * KG; k < (grp + 1) * KG; ++k) {
      double x[4], wv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) x[r] = sm.a[(tr + RQ * r) * WS + k];
#pragma unroll
      for (int i = 0; i < 4; ++i) wv[i] = sm.w[(tc + 16 * i) * WS + k];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[r][i] += x[r] * wv[i];
    }
    double* P = sm.dh + (size_t)grp * MS * HS;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int i = 0; i < 4; ++i) P[(tr + RQ * r) * HS + tc + 16 * i] = acc[r][i];
  }
  __syncthreads();
  for (int o = tid; o < MS * HID; o += NT) {
    const int s = o >> 6, j = o & 63;
    double v = 0.0;
#pragma unroll
    for (int g = 0; g < NG; ++g) v += sm.dh[(size_t)g * MS * HS + s * HS + j];
    sm.hpart[s * HS + j] = v;                         // hpart == P_{64 / MS}: every element is read before it is rewritten
  }
  stamp(prof, 5, tid);
  cluster_sync();                                        // #1: all six partial H are in shared memory
  stamp(prof, 6, tid);
  if (c == 0 && tid == 0 && a.calls != nullptr) {
    if (a.arrive == nullptr || nsplit == 1) a.calls[l] = call + 1;
    else if (atomicAdd(a.arrive + l, 1u) == (unsigned)nsplit - 1) { a.arrive[l] = 0; a.calls[l] = call + 1; }
  }

  // ---- reduce-scatter of H + fc2 / loss / their backward for this CTA's samples --------------------------------------------
  const int s0 = own_lo(c), ns = own_lo(c + 1) - s0;
  const double inv_bs = 1.0 / (double)(bg.bs ? bg.bs : 1);
  for (int o = tid; o < ns * HID; o += NT) {
    const int sl = o >> 6, j = o & 63;
    const double* src = sm.hpart + (s0 + sl) * HS + j;
    double v = sm.b1[j];
#pragma unroll
    for (int r = 0; r < CL; ++r) v += ld_dsmem(map_to(src, (uint32_t)r));
    sm.h_loc[o] = v > 0.0 ? v : 0.0;
  }
  __syncthreads();
  {
    const int o = tid >> 2, part = tid & 3;              // 4 lanes per logit
    const bool live = o < ns * NCLS;
    const int sl = live ? o / NCLS : 0, cc = live ? o - sl * NCLS : 0;
    double v = 0.0;
    if (live) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) { const int j = part * 16 + jj; v += sm.h_loc[sl * HID + j] * sm.w2[cc * HID + j]; }
    }
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (live && part == 0) sm.z[sl * 16 + cc] = v + sm.b2[cc];
  }
  __syncthreads();
  if (warp < ns) {                                       // log-softmax + NLL: one warp per sample, one lane per class
    const int sl = warp, s = s0 + sl;
    const bool cls = lane < NCLS;
    const double zc = cls ? sm.z[sl * 16 + lane] : -1.0e300;
    const double mx = wmax(zc);
    const double se = wsum(cls ? exp(zc - mx) : 0.0);
    const double lse = mx + log(se);
    const int y = sm.label[s];
    const double ok = (double)sm.valid[s];
    if (cls) sm.dz[sl * 16 + lane] = ok * inv_bs * (exp(zc - lse) - (lane == y ? 1.0 : 0.0));
    if (lane == y) sm.red[sl] = ok * (lse - zc);
  }
  __syncthreads();
  for (int o = tid; o < ns * HID; o += NT) {
    const int sl = o >> 6, j = o & 63;
    double v = 0.0;
#pragma unroll
    for (int cc = 0; cc < NCLS; ++cc) v += sm.dz[sl * 16 + cc] * sm.w2[cc * HID + j];
    sm.dh_loc[o] = sm.h_loc[o] > 0.0 ? v : 0.0;
  }
  __syncthreads();
  for (int o = tid; o < NCLS * HID; o += NT) {
    const int cc = o >> 6, j = o & 63;
    double v = 0.0;
    for (int sl = 0; sl < ns; ++sl) v += sm.dz[sl * 16 + cc] * sm.h_loc[sl * HID + j];
    sm.part[PART_W2 + o] = v;
  }
  if (tid < HID) {
    double v = 0.0;
    for (int sl = 0; sl < ns; ++sl) v += sm.dh_loc[sl * HID + tid];
    sm.part[PART_B1 + tid] = v;
  } else if (tid >= 64 && tid < 64 + NCLS) {
    double v = 0.0;
    for (int sl = 0; sl < ns; ++sl) v += sm.dz[sl * 16 + (tid - 64)];
    sm.part[PART_B2 + (tid - 64)] = v;
  } else if (tid == 96) {
    double v = 0.0;
    for (int sl = 0; sl < ns; ++sl) v += sm.red[sl];
    sm.part[PART_LOSS] = v * inv_bs;
  }
  stamp(prof, 7, tid);
  cluster_sync();                                        // #2: every owner's dH rows and fc2 / b1 / loss shares are final
  stamp(prof, 8, tid);
  double* gp = reinterpret_cast<double*>(a.grad_part) + ((size_t)l * nsplit + bsplit) * a.n_pad;
  // CTA c reduces its sixth of the fc2 / b1 / loss shares over the cluster (the peers stay resident until the last barrier)
  {
    constexpr int NE = PART_N - PART_B1, PER = (NE + CL - 1) / CL;
    const int o = PART_B1 + c * PER + tid;
    if (tid < PER && o < PART_N) {
      double v = 0.0;
#pragma unroll
      for (int r = 0; r < CL; ++r) v += ld_dsmem(map_to(sm.part + o, (uint32_t)r));
      if (o < PART_W2) gp[a.off_b1 + (o - PART_B1)] = v;
      else if (o < PART_B2) gp[a.off_w2 + (o - PART_W2)] = v;
      else if (o < PART_LOSS) gp[a.off_b2 + (o - PART_B2)] = v;
      else {
        a.loss_part[l * nsplit + bsplit] = (float)v;
        if (a.loss_mirror != nullptr) a.loss_mirror[l * nsplit + bsplit] = (float)v;
      }
    }
  }
  // ---- gather all MS dH rows from their owners ------------------------------------------------------------------------------
  for (int o = tid; o < MS * HID; o += NT) {
    const int s = o >> 6, j = o & 63;
    int r = 0;
#pragma unroll
    for (int q = 1; q < CL; ++q) r += (s >= own_lo(q)) ? 1 : 0;
    sm.dh[s * HS + j] = ld_dsmem(map_to(sm.dh_loc + (s - own_lo(r)) * HID + j, (uint32_t)r));
  }
  __syncthreads();
  stamp(prof, 9, tid);

  // ---- GEMM 2: da1_c[s][k] = sum_j dH[s][j] W[j][k]; tile 4 rows x 5 columns (k = tc + 16 i < 72).  With MS <= 32 the j range
  //      is split over two thread groups: group 1 parks its partial tile in the (dead) hpart rows, group 0 adds it -----------
  constexpr int NG2 = (MS <= 32) ? 2 : 1, JG = HID / NG2;
  double d2[4][5];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int i = 0; i < 5; ++i) d2[r][i] = 0.0;
  if (grp < NG2) {
#pragma unroll 2
    for (int j = grp * JG; j < (grp + 1) * JG; ++j) {
      double x[4], wv[5];
#pragma unroll
      for (int r = 0; r < 4; ++r) x[r] = sm.dh[(tr + RQ * r) * HS + j];
#pragma unroll
      for (int i = 0; i < 5; ++i) wv[i] = (tc + 16 * i < KC) ? sm.w[j * WS + tc + 16 * i] : 0.0;
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 5; ++i) d2[r][i] += x[r] * wv[i];
    }
    if (NG2 == 2 && grp == 1) {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 5; ++i)
          if (tc + 16 * i < KC) sm.hpart[(tr + RQ * r) * KC + tc + 16 * i] = d2[r][i];
    }
  }
  stamp(prof, 10, tid);
  // ---- GEMM 3: dW1_c[j][k] = sum_s dH[s][j] A[s][k]; tile 4 features (tr3 + 16 r) x 5 columns; 256 threads -----------------
  if (tid < 256) {
    const int tr3 = tid >> 4, tc3 = tid & 15;
    double d3[4][5];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int i = 0; i < 5; ++i) d3[r][i] = 0.0;
#pragma unroll 2
    for (int s = 0; s < MS; ++s) {
      double x[4], av[5];
#pragma unroll
      for (int r = 0; r < 4; ++r) x[r] = sm.dh[s * HS + tr3 + 16 * r];
#pragma unroll
      for (int i = 0; i < 5; ++i) av[i] = (tc3 + 16 * i < KC) ? sm.a[s * WS + tc3 + 16 * i] : 0.0;
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 5; ++i) d3[r][i] += x[r] * av[i];
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int k = tc3 + 16 * i;
      if (k < KC) {
        const int ch = k / CELLS, cell = k - ch * CELLS;
        double* g = gp + a.off_w1 + ch * NPOOL + CELLS * c + cell;
#pragma unroll
        for (int r = 0; r < 4; ++r) g[(size_t)(tr3 + 16 * r) * FC1_IN] = d3[r][i];
      }
    }
  }
  __syncthreads();      // every read of W (GEMM 2) and of A / dH (GEMM 3) is done; group 1's partial tile is parked
  stamp(prof, 11, tid);
  double* da1 = sm.w;   // W's rows become da1 [s][72], masked by ReLU'(a1)
  if (grp == 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const int s = tr + RQ * r, k = tc + 16 * i;
        if (k < KC) {
          const double v = d2[r][i] + (NG2 == 2 ? sm.hpart[s * KC + k] : 0.0);
          da1[s * KC + k] = (sm.arg[s * KC + k] & 4) ? v : 0.0;
        }
      }
  }
  __syncthreads();
  // ---- conv grads.  da1 is sparse (ReLU mask): (1) deterministic per-channel compaction of the non-zero (sample, cell)
  //      entries (ballot + prefix over 32-entry chunks, so the order — and the fp64 sums — never depend on timing);
  //      (2) five warps per channel walk that channel's dense list, each entry routes da1 to its argmax conv position;
  //      (3) ONE fold over lane pairs + transposition through the dead A / dH tiles for all three channels --------------
  constexpr int NI = MS * CELLS, NCH = NI / 32, CGW = 5, CGT = CGW * 32;     // entries / chunks per channel; warps / threads per channel
  static_assert(F * CGW <= NT / 32 && NI % 32 == 0 && NI <= 2048, "conv-grad work split");
  unsigned short* list = reinterpret_cast<unsigned short*>(sm.hpart);      // [F][NI] (hpart is dead: group 1's partial was consumed)
  int* ccount = reinterpret_cast<int*>(list + F * NI);                     // [F * NCH] chunk counts, then [F] totals
  static_assert(sizeof(unsigned short) * F * NI + sizeof(int) * (F * NCH + F) <= sizeof(double) * 64 * HS, "lists fit hpart");
  for (int q = warp; q < F * NCH; q += NT / 32) {
    const int ch = q / NCH, it = (q - ch * NCH) * 32 + lane;
    const int s = it / CELLS, cell = it - s * CELLS;
    const unsigned b = __ballot_sync(0xffffffffu, da1[s * KC + ch * CELLS + cell] != 0.0);
    if (lane == 0) ccount[q] = __popc(b);
  }
  __syncthreads();
  for (int q = warp; q < F * NCH; q += NT / 32) {
    const int ch = q / NCH, qq = q - ch * NCH, it = qq * 32 + lane;
    const int s = it / CELLS, cell = it - s * CELLS;
    int pre = 0;
    for (int j = lane; j < qq; j += 32) pre += ccount[ch * NCH + j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) pre += __shfl_xor_sync(0xffffffffu, pre, o);
    const bool nz = da1[s * KC + ch * CELLS + cell] != 0.0;
    const unsigned b = __ballot_sync(0xffffffffu, nz);
    if (nz) list[ch * NI + pre + __popc(b & ((1u << lane) - 1u))] =
        (unsigned short)(it | ((sm.arg[s * KC + ch * CELLS + cell] & 3) << 11));
    if (qq == NCH - 1 && lane == 0) ccount[F * NCH + ch] = pre + __popc(b);
  }
  __syncthreads();
  double* scratch = sm.a;                                                   // [F * 26][CGT / 2]
  static_assert(sizeof(double) * F * 26 * (CGT / 2) <= sizeof(double) * (64 * WS + 64 * HS), "conv-grad scratch fits A + dH");
  {
    const int gch = warp / CGW, tl = tid - gch * CGT;
    if (gch < F) {
      double cacc[26];
#pragma unroll
      for (int i = 0; i < 26; ++i) cacc[i] = 0.0;
      const int n = ccount[F * NCH + gch];
      for (int j = tl; j < n; j += CGT) {
        const unsigned e = list[gch * NI + j];
        const int it = e & 2047, ai = e >> 11;
        const int s = it / CELLS, cell = it - s * CELLS;
        const double g = da1[s * KC + gch * CELLS + cell];
        const int pr = cell / PHW, px = cell - pr * PHW;
        const PT* src = img + s * 224 + (2 * pr + (ai >> 1)) * HW + 2 * px + (ai & 1);
#pragma unroll
        for (int ky = 0; ky < KS; ++ky)
#pragma unroll
          for (int kx = 0; kx < KS; ++kx) cacc[ky * 5 + kx] += g * pix(src[ky * HW + kx]);
        cacc[25] += g;
      }
#pragma unroll
      for (int i = 0; i < 26; ++i) {
        const double v = cacc[i] + __shfl_xor_sync(0xffffffffu, cacc[i], 1);
        if ((lane & 1) == 0) scratch[(gch * 26 + i) * (CGT / 2) + (tl >> 1)] = v;
      }
    }
  }
  __syncthreads();
  for (int o = warp; o < F * 26; o += NT / 32) {
    double v = 0.0;
    for (int q = lane; q < CGT / 2; q += 32) v += scratch[o * (CGT / 2) + q];
    v = wsum(v);
    const int ch = o / 26, i = o - ch * 26;
    // this CTA's share goes straight into rank 0's collection buffer (its h_loc rows, dead since barrier #2)
    if (lane == 0) st_dsmem(map_to(sm.h_loc + c * 80 + (i < 25 ? ch * 25 + i : 75 + ch), 0u), v);
  }
  stamp(prof, 12, tid);
  cluster_sync();                                        // #3: all six conv-gradient shares are in rank 0's buffer
  if (c == 0 && tid < 78) {
    double v = 0.0;
#pragma unroll
    for (int r = 0; r < CL; ++r) v += sm.h_loc[r * 80 + tid];
    gp[tid < 75 ? a.off_wc + tid : a.off_bc + (tid - 75)] = v;
  }
  stamp(prof, 13, tid);
}

template <int MS>
static cudaError_t launch_ms(const Args& a, const GenericShape& gs, cudaStream_t st) {
  static cudaError_t prep = cudaFuncSetAttribute(mnist_cl64_train_kernel<MS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
  if (prep != cudaSuccess) return prep;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(CL, 64 / MS, a.L); cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = sizeof(Smem); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  static const bool no_pdl = getenv("NNDT_NO_PDL") != nullptr;
  cfg.attrs = attr; cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, mnist_cl64_train_kernel<MS>, a, gs);
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

int cl64_max_active_clusters() {
  if (cudaFuncSetAttribute(cl64::mnist_cl64_train_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(cl64::Smem)) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cl64::CL, 1, 1); cfg.blockDim = dim3(cl64::NT); cfg.dynamicSmemBytes = sizeof(cl64::Smem);
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, cl64::mnist_cl64_train_kernel<64>, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

}  // namespace mnist
}  // namespace nndt
