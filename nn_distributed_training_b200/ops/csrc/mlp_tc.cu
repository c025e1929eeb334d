// Tensor-core implementation of the implicit-density MLPs (FourierNet and ReLU nets) for sm_90a.
//
// One CTA processes tiles of 128 batch rows.  Per tile the hidden GEMMs run on the tensor cores as warp-level
// mma.sync m16n8k16 bf16 x bf16 -> fp32: activations live in shared memory as bf16 slabs of [rows][64] (16-byte
// chunks XOR-swizzled by row & 7, so both row- and column-wise fragment loads are free of bank conflicts) that are
// written by the previous layer's epilogue, weights are staged once per CTA as bf16 slabs, and each warp keeps the
// fp32 accumulators of its 16-row block in registers for the fused bias+activation epilogue.  The K=2 Fourier/SIREN
// input layer (sin on the SFU) and the 64->1 output layer (+sigmoid, +loss) stay on CUDA cores inside the same kernel.
// Reference op chain: models/fourier_nn.py:33-35,48-57 driven by
// problems/dist_online_dense_problem.py:117-127 (5 eager GEMMs + elementwise kernels per pass).
#include <cuda_bf16.h>

#include "common.cuh"
#include "mlp.h"
#include "sampler.cuh"

namespace nndt {
namespace mlp {

constexpr int NT = 256;         // forward CTA: 8 warps x 16 rows of the tile
constexpr int TILE = 128;
constexpr int HID = 64;
constexpr int MAX_DIN = 4;
constexpr int ROW_BYTES = 128;                   // 64 bf16
constexpr int ACT_SLAB = TILE * ROW_BYTES;       // 16 KB: 128 rows x 64 bf16
constexpr int W_SLAB = HID * ROW_BYTES;          // 8 KB: 64 rows x 64 bf16

// byte offset of the 16-byte chunk `chunk` (0..7) of row `row` inside a swizzled slab
NNDT_DEVINL uint32_t swz_chunk_off(int row, int chunk) {
  return (uint32_t)row * ROW_BYTES + (uint32_t)((chunk ^ (row & 7)) << 4);
}
// byte offset of element `col` (0..63) of row `row`
NNDT_DEVINL uint32_t swz_off(int row, int col) { return swz_chunk_off(row, col >> 3) + (uint32_t)(col & 7) * 2u; }

// pack 8 fp32 -> 8 bf16 (16 bytes)
NNDT_DEVINL uint4 pack_bf16x8(const float* v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]);
  __nv_bfloat162 b = __floats2bfloat162_rn(v[2], v[3]);
  __nv_bfloat162 c = __floats2bfloat162_rn(v[4], v[5]);
  __nv_bfloat162 d = __floats2bfloat162_rn(v[6], v[7]);
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&a);
  o.y = *reinterpret_cast<uint32_t*>(&b);
  o.z = *reinterpret_cast<uint32_t*>(&c);
  o.w = *reinterpret_cast<uint32_t*>(&d);
  return o;
}
NNDT_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&p);
}

// ---- operand fragments -----------------------------------------------------------------------------------------
// Elements (row, k) and (row, k + 1) of slabs [rows][64] laid `stride` bytes apart along k (k even): one 32-bit load.
NNDT_DEVINL uint32_t ld_k(const uint8_t* s, int stride, int row, int k) {
  return *reinterpret_cast<const uint32_t*>(s + (k >> 6) * stride + swz_off(row, k & 63));
}
// Elements (k, col) and (k + 1, col) of slabs [k rows][64 cols] laid `stride` bytes apart along col: the transposed
// reading of the same tiles (backward GEMMs need no transposed copies).
NNDT_DEVINL uint32_t ld_mn(const uint8_t* s, int stride, int k, int col) {
  const uint8_t* p = s + (col >> 6) * stride;
  const uint32_t lo = *reinterpret_cast<const uint16_t*>(p + swz_off(k, col & 63));
  const uint32_t hi = *reinterpret_cast<const uint16_t*>(p + swz_off(k + 1, col & 63));
  return lo | (hi << 16);
}

NNDT_DEVINL void mma_bf16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// c[j] = sum_k A(m0 + ., k) B(k, n0 + 8 j + .) over `ksteps` steps of 16 for NJ adjacent 16 x 8 tiles.  `A(m, k)` and
// `B(k, n)` return the packed pairs (k, k + 1).  Fragment coordinates (g = lane >> 2, t = lane & 3):
//   c0 (g, 2t)  c1 (g, 2t+1)  c2 (g+8, 2t)  c3 (g+8, 2t+1)
template <int NJ, class FA, class FB>
NNDT_DEVINL void gemm_tiles(float (&c)[NJ][4], int m0, int n0, int ksteps, int lane, FA A, FB B) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < NJ; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
#pragma unroll 1
  for (int ks = 0; ks < ksteps; ++ks) {
    const int k = 16 * ks + 2 * t;
    const uint32_t a[4] = {A(m0 + g, k), A(m0 + g + 8, k), A(m0 + g, k + 8), A(m0 + g + 8, k + 8)};
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const uint32_t b[2] = {B(k, n0 + 8 * j + g), B(k + 8, n0 + 8 * j + g)};
      mma_bf16(c[j], a, b);
    }
  }
}

// epilogue of a hidden layer for NJ tiles at (m0, n0): h = relu(acc + bias) (kept in acc) -> bf16 pairs of `dst`
template <int NJ>
NNDT_DEVINL void hidden_epilogue(float (&c)[NJ][4], int m0, int n0, const float* bias, uint8_t* dst, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = n0 + 8 * j + 2 * t;
#pragma unroll
    for (int i = 0; i < 4; ++i) c[j][i] = fmaxf(c[j][i] + bias[col + (i & 1)], 0.f);
    if (dst != nullptr) {
      *reinterpret_cast<uint32_t*>(dst + swz_off(m0 + g, col)) = pack_bf16x2(c[j][0], c[j][1]);
      *reinterpret_cast<uint32_t*>(dst + swz_off(m0 + g + 8, col)) = pack_bf16x2(c[j][2], c[j][3]);
    }
  }
}

template <int H1>
struct FwdSmem {
  alignas(16) uint8_t w1[(H1 / 64) * W_SLAB];
  alignas(16) uint8_t w2[W_SLAB];
  alignas(16) uint8_t w3[W_SLAB];
  alignas(16) uint8_t h1[(H1 / 64) * ACT_SLAB];
  alignas(16) uint8_t ha[ACT_SLAB];
  alignas(16) uint8_t hb[ACT_SLAB];
  float w0[H1 * MAX_DIN];
  float b0[H1];
  float b1[HID], b2[HID], b3[HID], w4[HID];
  float b4;
  float xs[TILE * MAX_DIN];
};

// stage a [64 x K] fp32 weight matrix (row-major, K multiple of 64) as K/64 bf16 swizzled slabs
template <int TN>
NNDT_DEVINL void stage_weight(uint8_t* dst, const float* w, int K, int tid) {
  const int chunks = HID * (K / 8);            // 16-byte chunks
  for (int o = tid; o < chunks; o += TN) {
    const int n = o / (K / 8), c = o - n * (K / 8);
    const float4 lo = *reinterpret_cast<const float4*>(w + (size_t)n * K + 8 * c);
    const float4 hi = *reinterpret_cast<const float4*>(w + (size_t)n * K + 8 * c + 4);
    const float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    const int slab = c >> 3, cc = c & 7;
    *reinterpret_cast<uint4*>(dst + slab * W_SLAB + swz_chunk_off(n, cc)) = pack_bf16x8(v);
  }
}

template <int H1, int TN, class S>
NNDT_DEVINL void stage_all_weights(S& sm, const Args& a, const float* th, int tid) {
  stage_weight<TN>(sm.w1, th + a.off[2], H1, tid);
  stage_weight<TN>(sm.w2, th + a.off[4], HID, tid);
  stage_weight<TN>(sm.w3, th + a.off[6], HID, tid);
  for (int o = tid; o < H1 * a.d_in; o += TN) sm.w0[o] = th[a.off[0] + o];
  for (int o = tid; o < H1; o += TN) sm.b0[o] = th[a.off[1] + o];
  if (tid < HID) {
    sm.b1[tid] = th[a.off[3] + tid];
    sm.b2[tid] = th[a.off[5] + tid];
    sm.b3[tid] = th[a.off[7] + tid];
    sm.w4[tid] = th[a.off[8] + tid];
  }
  if (tid == 0) sm.b4 = th[a.off[9]];
}

// first layer on CUDA cores: h1[r][f] = relu(sin(scale * z)) or relu(z), z = x[r] . W0[f] + b0[f]
template <int H1, int DIN, int TN, class S>
NNDT_DEVINL void first_layer(S& sm, const Args& a, int tid) {
  const int r = tid & (TILE - 1);
  const int half = tid >> 7;                       // TN/128 thread groups split the features
  float x[DIN];
#pragma unroll
  for (int d = 0; d < DIN; ++d) x[d] = sm.xs[r * MAX_DIN + d];
  constexpr int CH = H1 / 8 / (TN / TILE);         // 16-byte chunks per thread
  for (int c = 0; c < CH; ++c) {
    const int chunk = half * CH + c;               // global chunk index along the H1 features
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int f = chunk * 8 + e;
      float z = sm.b0[f];
#pragma unroll
      for (int d = 0; d < DIN; ++d) z = fmaf(x[d], sm.w0[f * DIN + d], z);
      if (a.first_act == kFirstSinRelu) z = __sinf(a.scale * z);
      v[e] = fmaxf(z, 0.f);
    }
    const int slab = chunk >> 3, cc = chunk & 7;
    *reinterpret_cast<uint4*>(sm.h1 + slab * ACT_SLAB + swz_chunk_off(r, cc)) = pack_bf16x8(v);
  }
}

template <int H1, int DIN>
__global__ void __launch_bounds__(NT, 1) mlp_forward_kernel(const Args a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  FwdSmem<H1>& sm = *reinterpret_cast<FwdSmem<H1>*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int l = blockIdx.y;
  const float* th = a.theta + (size_t)l * a.n_pad;
  const int m0 = 16 * warp;                        // this warp's 16 rows of the tile, all 64 columns

  stage_all_weights<H1, NT>(sm, a, th, tid);
  __syncthreads();
  auto wk = [](const uint8_t* w) { return [w](int k, int n) { return ld_k(w, W_SLAB, n, k); }; };
  auto hk = [](const uint8_t* h) { return [h](int m, int k) { return ld_k(h, ACT_SLAB, m, k); }; };

  const int ntiles = (a.n_rows + TILE - 1) / TILE;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int row0 = tile * TILE;
    for (int o = tid; o < TILE * a.d_in; o += NT) {
      const int r = o / a.d_in, d = o - r * a.d_in;
      sm.xs[r * MAX_DIN + d] = (row0 + r < a.n_rows) ? a.x[(size_t)(row0 + r) * a.d_in + d] : 0.f;
    }
    __syncthreads();
    first_layer<H1, DIN, NT>(sm, a, tid);
    __syncthreads();

    // a warp reads only its own 16 rows of the activations, which it wrote itself: the hidden layers need no CTA barrier
    float c[8][4];
    gemm_tiles<8>(c, m0, 0, H1 / 16, lane, hk(sm.h1), wk(sm.w1));
    hidden_epilogue<8>(c, m0, 0, sm.b1, sm.ha, lane);
    __syncwarp();
    gemm_tiles<8>(c, m0, 0, HID / 16, lane, hk(sm.ha), wk(sm.w2));
    hidden_epilogue<8>(c, m0, 0, sm.b2, sm.hb, lane);
    __syncwarp();
    gemm_tiles<8>(c, m0, 0, HID / 16, lane, hk(sm.hb), wk(sm.w3));
    hidden_epilogue<8>(c, m0, 0, sm.b3, nullptr, lane);
    // ---- output layer ------------------------------------------------------------------------------------------
    float dot[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + 2 * t;
      dot[0] = fmaf(c[j][0], sm.w4[col], fmaf(c[j][1], sm.w4[col + 1], dot[0]));
      dot[1] = fmaf(c[j][2], sm.w4[col], fmaf(c[j][3], sm.w4[col + 1], dot[1]));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      dot[h] += __shfl_xor_sync(0xffffffffu, dot[h], 1);
      dot[h] += __shfl_xor_sync(0xffffffffu, dot[h], 2);
    }
    if (t == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0 + g + 8 * h;
        if (row0 + row < a.n_rows) {
          float z = dot[h] + sm.b4;
          if (a.last_act == kLastSigmoid) z = 1.f / (1.f + __expf(-z));
          a.out[(size_t)l * a.n_rows + row0 + row] = z;
        }
      }
    }
    __syncthreads();
  }
}

template <int H1>
static cudaError_t launch_forward_t(const Args& a, int ctas, cudaStream_t st) {
  const int smem = (int)sizeof(FwdSmem<H1>);
  static cudaError_t attr = cudaFuncSetAttribute(mlp_forward_kernel<H1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (attr != cudaSuccess) return attr;
  if (a.d_in != 2) return cudaErrorInvalidValue;
  mlp_forward_kernel<H1, 2><<<dim3(ctas, a.L), NT, smem, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_forward(const Args& a, int ctas_per_node, cudaStream_t st) {
  if (a.d_in > MAX_DIN) return cudaErrorInvalidValue;
  switch (a.h1) {
    case 64: return launch_forward_t<64>(a, ctas_per_node, st);
    case 128: return launch_forward_t<128>(a, ctas_per_node, st);
    case 256: return launch_forward_t<256>(a, ctas_per_node, st);
    default: return cudaErrorInvalidValue;
  }
}

// =====================================================================================
// Training: forward + backward of one minibatch per node, gradients to per-CTA partial rows.
//
// Backward GEMMs read the forward operand tiles transposed (ld_mn), so no transposed copies are made:
//   dH_{l-1}[128 x K_in] = dZ_l[128 x 64] . W_l
//   dW_l                 = dZ_l^T . H_{l-1}, K = the 128 batch rows of the tile
//   bias / first-layer grads = dZ^T . [x, 1]: the same GEMM against an 8-column tile holding the rows' inputs and a
//                          ones column, so no cross-lane shuffle reductions are needed.
// The weight gradients of a tile are added into this CTA's partial row of the node (the first tile stores); every
// element is owned by one thread, so the read-modify-write needs no atomics.
// =====================================================================================
constexpr int NTT = 512;       // training CTA: 16 warps = 8 row blocks of 16 x 2 column halves of 32

template <int H1>
struct TrainSmem {
  alignas(16) uint8_t w1[(H1 / 64) * W_SLAB];
  alignas(16) uint8_t w2[W_SLAB];
  alignas(16) uint8_t w3[W_SLAB];
  alignas(16) uint8_t h1[(H1 / 64) * ACT_SLAB];   // h1, later dZ1
  alignas(16) uint8_t dz[ACT_SLAB];               // dZ of the layer being back-propagated
  alignas(16) uint8_t h2[ACT_SLAB];
  alignas(16) uint8_t h3[ACT_SLAB];
  alignas(16) __nv_bfloat16 xa[TILE * 8];         // [x_0..x_{DIN-1}, 1, 0...] per row
  float w0[H1 * MAX_DIN];
  float b0[H1];
  float b1[HID], b2[HID], b3[HID], w4[HID];
  float b4;
  float g_w4[HID];
  float g_b4;
  float loss_acc;
  float xs[TILE * MAX_DIN];
  float ys[TILE];
  float part[2 * TILE];
  float dz5[TILE];
  int ridx[TILE];
};

NNDT_DEVINL void acc_store(float* p, float v, bool add) { *p = add ? *p + v : v; }

// grad[m][n] (+)= sum_r A[r][m] B[r][n] over the 128 tile rows for the M x 64 weight gradients (M = 64 or H1);
// A: slabs [128 rows][64] `a_stride` apart along m, B: one slab [128 rows][64].  Output element (m, n) goes to
// dst[m * ms + n * ns].
NNDT_DEVINL void weight_grad(const uint8_t* A, int a_stride, const uint8_t* B, int M, float* dst, int ms, int ns,
                             bool add, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  for (int tile = warp; tile < (M / 16) * 8; tile += NTT / 32) {
    const int m0 = 16 * (tile >> 3), n0 = 8 * (tile & 7);
    float c[1][4];
    gemm_tiles<1>(c, m0, n0, TILE / 16, lane, [A, a_stride](int m, int k) { return ld_mn(A, a_stride, k, m); },
                  [B](int k, int n) { return ld_mn(B, ACT_SLAB, k, n); });
#pragma unroll
    for (int i = 0; i < 4; ++i) acc_store(dst + (m0 + g + 8 * (i >> 1)) * ms + (n0 + 2 * t + (i & 1)) * ns, c[0][i], add);
  }
}

// sum_r A[r][m] [x, 1][r][n] for the M features of A: n < DIN goes to w_dst[m * DIN + n] (unless null), n == DIN to
// b_dst[m]
template <int DIN>
NNDT_DEVINL void input_grad(const uint8_t* A, int M, const __nv_bfloat16* xa, float* w_dst, float* b_dst, bool add,
                            int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const uint16_t* xu = reinterpret_cast<const uint16_t*>(xa);
  for (int tile = warp; tile < M / 16; tile += NTT / 32) {
    const int m0 = 16 * tile;
    float c[1][4];
    gemm_tiles<1>(c, m0, 0, TILE / 16, lane, [A](int m, int k) { return ld_mn(A, ACT_SLAB, k, m); },
                  [xu](int k, int n) { return (uint32_t)xu[k * 8 + n] | ((uint32_t)xu[(k + 1) * 8 + n] << 16); });
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + g + 8 * (i >> 1), n = 2 * t + (i & 1);
      if (n < DIN && w_dst != nullptr) acc_store(w_dst + m * DIN + n, c[0][i], add);
      else if (n == DIN) acc_store(b_dst + m, c[0][i], add);
    }
  }
}

template <int H1, int DIN>
__global__ void __launch_bounds__(NTT, 1) mlp_train_kernel(const Args a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  TrainSmem<H1>& sm = *reinterpret_cast<TrainSmem<H1>*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int m0 = 16 * (warp & 7), nb = 32 * (warp >> 3);     // this warp's 16 rows x 32 columns of a 64-wide layer

  // ---- static work partition: items (node, tile) in node-major order -------------------------
  const int Tmax = (a.batch + TILE - 1) / TILE;
  const int I = a.L * Tmax, G = gridDim.x, c = blockIdx.x;
  const int it0 = (int)(((long long)c * I) / G), it1 = (int)(((long long)(c + 1) * I) / G);

  int cur = -1;          // node whose weights are staged
  bool have_acc = false; // this CTA's partial row of node `cur` holds the gradients of at least one tile
  float* gp = nullptr;   // that partial row
  int slot = 0;
  uint32_t bs = 0;
  NodeStream ns{};                     // the current node's batch draws (unless direct)
  auto wk = [](const uint8_t* w) { return [w](int k, int n) { return ld_k(w, W_SLAB, n, k); }; };
  auto hk = [](const uint8_t* h) { return [h](int mm, int k) { return ld_k(h, ACT_SLAB, mm, k); }; };

  for (int it = it0; it <= it1; ++it) {
    const int l = (it < it1) ? it / Tmax : -1;
    if (l != cur) {
      // ---------------- flush the finished node segment ---------------------------------------
      if (cur >= 0) {
        if (!have_acc) {       // no tile of the node had rows for this CTA: its GEMM-derived gradients are zero
          for (int o = tid; o < HID * HID; o += NTT) { gp[a.off[6] + o] = 0.f; gp[a.off[4] + o] = 0.f; }
          for (int o = tid; o < HID * H1; o += NTT) gp[a.off[2] + o] = 0.f;
          for (int o = tid; o < H1 * DIN; o += NTT) gp[a.off[0] + o] = 0.f;
          for (int o = tid; o < H1; o += NTT) gp[a.off[1] + o] = 0.f;
          if (tid < HID) { gp[a.off[7] + tid] = 0.f; gp[a.off[5] + tid] = 0.f; gp[a.off[3] + tid] = 0.f; }
        }
        if (tid < HID) gp[a.off[8] + tid] = sm.g_w4[tid];
        if (tid == 0) { gp[a.off[9]] = sm.g_b4; a.loss_part[cur * a.S + slot] = sm.loss_acc; }
        __syncthreads();
      }
      if (l < 0) break;
      // ---------------- set up the next node ----------------------------------------------------
      cur = l;
      have_acc = false;
      {
        const long long first_item = (long long)l * Tmax;
        int cf = (int)((first_item * G) / I);
        while ((long long)(cf + 1) * I / G <= first_item) ++cf;
        while ((long long)cf * I / G > first_item) --cf;
        slot = c - cf;         // this CTA's slot among the CTAs that cover node l
        gp = a.grad_part + ((size_t)l * a.S + slot) * a.n_pad;
      }
      const float* th = a.theta + (size_t)l * a.n_pad;
      stage_all_weights<H1, NTT>(sm, a, th, tid);
      if (tid < HID) sm.g_w4[tid] = 0.f;
      if (tid == 0) { sm.g_b4 = 0.f; sm.loss_acc = 0.f; }
      if (a.direct) {
        bs = (uint32_t)a.batch;
      } else {
        const long long* wt = a.win_table != nullptr
                                  ? reinterpret_cast<const long long*>(a.win_table) + (size_t)l * kWinTableLen : nullptr;
        ns = node_stream((uint32_t)a.calls[l], (uint32_t)a.shard_len[l], (uint32_t)a.batch, (uint32_t)a.seed,
                         (uint32_t)(a.node0 + l), a.shard_off[l], wt);
        bs = ns.size;
      }
      __syncthreads();
    }
    const int tile = it - l * Tmax;
    const uint32_t t0 = (uint32_t)tile * TILE;
    if (t0 >= bs) continue;                              // partial batch: nothing in this tile
    const float inv_bs = 1.f / (float)bs;

    // ---- gather the tile's rows ------------------------------------------------------------------------
    if (tid < TILE) {
      int my_idx = -1;
      const uint32_t tt = t0 + tid;
      if (tt < bs) {
        my_idx = a.direct ? (int)(l * a.batch + tt) : stream_row(ns, tt);
      }
      sm.ridx[tid] = my_idx;
      sm.ys[tid] = my_idx >= 0 ? a.y[my_idx] : 0.f;
      float xv[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) xv[e] = 0.f;
#pragma unroll
      for (int d = 0; d < DIN; ++d) {
        xv[d] = my_idx >= 0 ? a.x[(size_t)my_idx * DIN + d] : 0.f;
        sm.xs[tid * MAX_DIN + d] = xv[d];
      }
      xv[DIN] = my_idx >= 0 ? 1.f : 0.f;
      *reinterpret_cast<uint4*>(sm.xa + tid * 8) = pack_bf16x8(xv);
    }
    __syncthreads();
    first_layer<H1, DIN, NTT>(sm, a, tid);
    __syncthreads();

    // ======================= forward ===============================================================
    float acc[4][4];
    gemm_tiles<4>(acc, m0, nb, H1 / 16, lane, hk(sm.h1), wk(sm.w1));
    hidden_epilogue<4>(acc, m0, nb, sm.b1, sm.h2, lane);
    __syncthreads();
    gemm_tiles<4>(acc, m0, nb, HID / 16, lane, hk(sm.h2), wk(sm.w2));
    hidden_epilogue<4>(acc, m0, nb, sm.b2, sm.h3, lane);
    __syncthreads();
    gemm_tiles<4>(acc, m0, nb, HID / 16, lane, hk(sm.h3), wk(sm.w3));
    hidden_epilogue<4>(acc, m0, nb, sm.b3, nullptr, lane);     // acc = h4[m0 + ..][nb + ..]
    // ---- output layer, loss, dL/dz5 --------------------------------------------------------------------
    {
      float dot[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = nb + 8 * j + 2 * t;
        dot[0] = fmaf(acc[j][0], sm.w4[col], fmaf(acc[j][1], sm.w4[col + 1], dot[0]));
        dot[1] = fmaf(acc[j][2], sm.w4[col], fmaf(acc[j][3], sm.w4[col + 1], dot[1]));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        dot[h] += __shfl_xor_sync(0xffffffffu, dot[h], 1);
        dot[h] += __shfl_xor_sync(0xffffffffu, dot[h], 2);
        if (t == 0) sm.part[(warp >> 3) * TILE + m0 + g + 8 * h] = dot[h];
      }
      __syncthreads();
      if (tid < TILE) {
        const int row = tid;
        const bool valid = sm.ridx[row] >= 0;
        const float z = sm.part[row] + sm.part[TILE + row] + sm.b4;
        const float y = sm.ys[row];
        float p = z, dpdz = 1.f;
        if (a.last_act == kLastSigmoid) { p = 1.f / (1.f + __expf(-z)); dpdz = p * (1.f - p); }
        float loss, gz;
        if (a.loss == kLossBCE) {
          loss = -(y * fmaxf(__logf(p), -100.f) + (1.f - y) * fmaxf(__logf(1.f - p), -100.f));
          gz = (a.last_act == kLastSigmoid) ? (p - y) : (p - y) / fmaxf(p * (1.f - p), 1e-12f);
        } else if (a.loss == kLossMSE) {
          loss = (p - y) * (p - y); gz = 2.f * (p - y) * dpdz;
        } else {
          loss = fabsf(p - y); gz = (p > y ? 1.f : (p < y ? -1.f : 0.f)) * dpdz;
        }
        sm.dz5[row] = valid ? gz * inv_bs : 0.f;
        const float lsum = warp_sum(valid ? loss * inv_bs : 0.f);
        const float gsum = warp_sum(valid ? gz * inv_bs : 0.f);
        if (lane == 0) { atomicAdd(&sm.loss_acc, lsum); atomicAdd(&sm.g_b4, gsum); }
      }
      __syncthreads();
    }
    // ======================= backward ================================================================
    {
      // layer 5 -> dz4 = dz5 * w4 * relu'(h4);  dW4 += dz5 * h4 (the one remaining shuffle reduction)
      const float d5[2] = {sm.dz5[m0 + g], sm.dz5[m0 + g + 8]};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = nb + 8 * j + 2 * t;
        float gw[2], dz[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) dz[i] = acc[j][i] > 0.f ? d5[i >> 1] * sm.w4[col + (i & 1)] : 0.f;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          gw[e] = fmaf(d5[0], acc[j][e], d5[1] * acc[j][2 + e]);
          gw[e] += __shfl_xor_sync(0xffffffffu, gw[e], 4);
          gw[e] += __shfl_xor_sync(0xffffffffu, gw[e], 8);
          gw[e] += __shfl_xor_sync(0xffffffffu, gw[e], 16);
        }
        if (g == 0) { atomicAdd(&sm.g_w4[col], gw[0]); atomicAdd(&sm.g_w4[col + 1], gw[1]); }
        *reinterpret_cast<uint32_t*>(sm.dz + swz_off(m0 + g, col)) = pack_bf16x2(dz[0], dz[1]);
        *reinterpret_cast<uint32_t*>(sm.dz + swz_off(m0 + g + 8, col)) = pack_bf16x2(dz[2], dz[3]);
      }
    }
    __syncthreads();
    // hidden layers 4 -> 3 -> 2: dW_l += dz_l^T . h_{l-1}; db_l += dz_l^T . [x,1]; dz_{l-1} = (dz_l . W_l) * relu'(h_{l-1})
#pragma unroll 1
    for (int layer = 3; layer >= 2; --layer) {
      const uint8_t* hs = layer == 3 ? sm.h3 : sm.h2;
      const uint8_t* w = layer == 3 ? sm.w3 : sm.w2;
      weight_grad(sm.dz, ACT_SLAB, hs, HID, gp + a.off[layer == 3 ? 6 : 4], HID, 1, have_acc, warp, lane);
      input_grad<DIN>(sm.dz, HID, sm.xa, nullptr, gp + a.off[layer == 3 ? 7 : 5], have_acc, warp, lane);
      gemm_tiles<4>(acc, m0, nb, HID / 16, lane, hk(sm.dz), [w](int k, int n) { return ld_mn(w, W_SLAB, k, n); });
      __syncthreads();                                   // every warp is done reading dz_l
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = nb + 8 * j + 2 * t;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + g + 8 * h;
          const __nv_bfloat162 hv = *reinterpret_cast<const __nv_bfloat162*>(hs + swz_off(row, col));
          const float z0 = __bfloat162float(hv.x) > 0.f ? acc[j][2 * h] : 0.f;
          const float z1 = __bfloat162float(hv.y) > 0.f ? acc[j][2 * h + 1] : 0.f;
          *reinterpret_cast<uint32_t*>(sm.dz + swz_off(row, col)) = pack_bf16x2(z0, z1);
        }
      }
      __syncthreads();
    }
    // dW1 (stored [64 out][H1 in]) = dz2^T . h1 read as h1^T . dz2: M = the H1 input features
    weight_grad(sm.h1, ACT_SLAB, sm.dz, H1, gp + a.off[2], 1, H1, have_acc, warp, lane);
    input_grad<DIN>(sm.dz, HID, sm.xa, nullptr, gp + a.off[3], have_acc, warp, lane);
    __syncthreads();                                     // h1 is dead: dz1 goes over it
    // ---- first layer: dz1 = (dz2 . W1) * act'(z1), 64 features at a time; [dW0|db0] += dz1^T [x,1] ----------------
    {
      float x[2][DIN];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int d = 0; d < DIN; ++d) x[h][d] = sm.xs[(m0 + g + 8 * h) * MAX_DIN + d];
#pragma unroll 1
      for (int f64 = 0; f64 < H1; f64 += 64) {
        gemm_tiles<4>(acc, m0, f64 + nb, HID / 16, lane, hk(sm.dz), [&sm](int k, int n) { return ld_mn(sm.w1, W_SLAB, k, n); });
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int f0 = f64 + nb + 8 * j + 2 * t;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int f = f0 + (i & 1);
            float z = sm.b0[f];
#pragma unroll
            for (int d = 0; d < DIN; ++d) z = fmaf(x[i >> 1][d], sm.w0[f * DIN + d], z);
            float dact;
            if (a.first_act == kFirstSinRelu) {
              float sn, cs;
              __sincosf(a.scale * z, &sn, &cs);
              dact = sn > 0.f ? cs * a.scale : 0.f;
            } else {
              dact = z > 0.f ? 1.f : 0.f;
            }
            acc[j][i] *= dact;
          }
          uint8_t* slab = sm.h1 + (f0 >> 6) * ACT_SLAB;
          *reinterpret_cast<uint32_t*>(slab + swz_off(m0 + g, f0 & 63)) = pack_bf16x2(acc[j][0], acc[j][1]);
          *reinterpret_cast<uint32_t*>(slab + swz_off(m0 + g + 8, f0 & 63)) = pack_bf16x2(acc[j][2], acc[j][3]);
        }
      }
      __syncthreads();
      for (int blk = 0; blk < H1 / 64; ++blk)
        input_grad<DIN>(sm.h1 + blk * ACT_SLAB, HID, sm.xa, gp + a.off[0] + blk * 64 * DIN, gp + a.off[1] + blk * 64,
                        have_acc, warp, lane);
    }
    have_acc = true;
    __syncthreads();                                     // the next tile overwrites xs / xa / h1
  }
}

template <int H1>
static cudaError_t launch_train_t(const Args& a, int ctas, cudaStream_t st) {
  const int smem = (int)sizeof(TrainSmem<H1>);
  static cudaError_t attr = cudaFuncSetAttribute(mlp_train_kernel<H1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (attr != cudaSuccess) return attr;
  if (a.d_in != 2) return cudaErrorInvalidValue;
  mlp_train_kernel<H1, 2><<<dim3(ctas), NTT, smem, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_train(const Args& a, int ctas, cudaStream_t st) {
  if (a.d_in > MAX_DIN) return cudaErrorInvalidValue;
  switch (a.h1) {
    case 64: return launch_train_t<64>(a, ctas, st);
    case 128: return launch_train_t<128>(a, ctas, st);
    case 256: return launch_train_t<256>(a, ctas, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace mlp
}  // namespace nndt
