// Device-side building blocks of the MNIST conv-net forward/backward (the batch-split kernel of mnist.cu).
#pragma once
#include "common.cuh"
#include "sampler.cuh"
#include "mnist.h"

namespace nndt {
namespace mnist {

constexpr int F = 3, KS = 5, HW = 28, PHW = 12, NPOOL = 144;
constexpr int FC1_IN = 432, HID = 64, NCLS = 10;
constexpr int W1_STRIDE = 436;          // padded fc1 row stride in smem (floats): conflict-free mma fragment loads
constexpr int A1_STRIDE = 436;          // same padding for the fc1 input rows (B / A fragments of the three GEMMs)
constexpr int KGROUPS = 6;              // fc1: the 54 k-steps of 8 are split over 6 warp groups
constexpr int XROW = 22;                // padded row stride of the even/odd column planes
constexpr int XPLANE = HW * XROW;       // 616 floats per plane
constexpr int CGROUP = 256;             // threads cooperating on one conv channel in the backward

// NT = 768 threads per CTA: 24 warps = 4 row tiles x 6 k-groups of the fc1-sized MMAs, >= 3 x CGROUP for the conv
// backward and >= FC1_IN for the element-wise phases.
template <int SPB, int NT>
struct Smem {
  float w1[HID * W1_STRIDE];            // fc1 weights; later scratch for the conv-grad reduce
  float xe[SPB * XPLANE];
  float xo[SPB * XPLANE];
  float a1[8 * A1_STRIDE];              // fc1 input [sample][k]; rows >= SPB stay zero (K / N padding of the MMAs)
  float da1[SPB * FC1_IN];
  float hpart[KGROUPS * 8 * HID];       // fc1 partial sums [k-group][sample][j]
  float h[SPB * HID];
  float dh[SPB * HID];
  float dhT[HID * 8];                   // [j][s], row padded to 8 samples -> two 128-bit broadcast loads
  float w2[NCLS * HID];
  float z[SPB * 16];
  float dz[SPB * 16];
  float wc[F * KS * KS + 4];
  float red[80];
  float b1[HID];
  float b2[16];
  int sidx[SPB];
  int label[SPB];
  float valid[SPB];
  unsigned char arg[SPB * FC1_IN];
  alignas(8) uint64_t w1_bar;           // TMA transaction barrier of the fc1 weight staging
};

// Pixel gather in two halves so other work can sit between the global loads and their first use:
// 196 groups of 4 pixels per sample; every global load of a thread is issued before the first conversion.
template <int SPB, int NT>
struct ImgRegs {
  static constexpr int PER = (SPB * 196 + NT - 1) / NT;
  uint32_t u8[PER];
  float4 f[PER];
};
template <int SPB, int NT>
__device__ __forceinline__ void issue_image_loads(const Smem<SPB, NT>& sm, const Args& a, int tid, ImgRegs<SPB, NT>& r) {
  constexpr int PER = ImgRegs<SPB, NT>::PER;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int o = tid + i * NT;
    r.u8[i] = 0; r.f[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (o < SPB * 196) {
      const int s = o / 196, q = o - s * 196;
      if (sm.valid[s] != 0.f) {
        const size_t base = (size_t)sm.sidx[s] * 784 + 4 * q;
        if (a.x_is_u8) r.u8[i] = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const unsigned char*>(a.x) + base);
        else r.f[i] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.x) + base);
      }
    }
  }
}
template <int SPB, int NT>
__device__ __forceinline__ void commit_images(Smem<SPB, NT>& sm, const Args& a, int tid, const ImgRegs<SPB, NT>& r) {
  constexpr int PER = ImgRegs<SPB, NT>::PER;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int o = tid + i * NT;
    if (o < SPB * 196) {
      const int s = o / 196, q = o - s * 196;
      const int row = (4 * q) / HW, col = (4 * q) - row * HW;
      float v0, v1, v2, v3;
      if (a.x_is_u8) {
        const bool ok = sm.valid[s] != 0.f;
        const uint32_t p = r.u8[i];
        v0 = ok ? ((p & 0xff) * (1.f / 255.f) - a.mean) * a.inv_std : 0.f;
        v1 = ok ? (((p >> 8) & 0xff) * (1.f / 255.f) - a.mean) * a.inv_std : 0.f;
        v2 = ok ? (((p >> 16) & 0xff) * (1.f / 255.f) - a.mean) * a.inv_std : 0.f;
        v3 = ok ? ((p >> 24) * (1.f / 255.f) - a.mean) * a.inv_std : 0.f;
      } else {
        v0 = r.f[i].x; v1 = r.f[i].y; v2 = r.f[i].z; v3 = r.f[i].w;
      }
      float* e = sm.xe + s * XPLANE + row * XROW + (col >> 1);
      float* d = sm.xo + s * XPLANE + row * XROW + (col >> 1);
      e[0] = v0; d[0] = v1; e[1] = v2; d[1] = v3;
    }
  }
}

template <int SPB, int NT>
__device__ __forceinline__ void conv_relu_pool(Smem<SPB, NT>& sm, int tid) {
  for (int it = tid; it < SPB * NPOOL; it += NT) {
    const int s = it / NPOOL, p = it - s * NPOOL;
    const int py = p / PHW, pxx = p - py * PHW;
    float patch[6][6];
    const float* e = sm.xe + s * XPLANE + (2 * py) * XROW + pxx;
    const float* o = sm.xo + s * XPLANE + (2 * py) * XROW + pxx;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        patch[r][2 * c] = e[r * XROW + c];
        patch[r][2 * c + 1] = o[r * XROW + c];
      }
    }
#pragma unroll
    for (int c = 0; c < F; ++c) {
      float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const float w = sm.wc[c * 25 + ky * 5 + kx];
          acc[0][0] = fmaf(w, patch[ky][kx], acc[0][0]);
          acc[0][1] = fmaf(w, patch[ky][kx + 1], acc[0][1]);
          acc[1][0] = fmaf(w, patch[ky + 1][kx], acc[1][0]);
          acc[1][1] = fmaf(w, patch[ky + 1][kx + 1], acc[1][1]);
        }
      }
      // first maximum wins, like ATen's max_pool2d
      float m = acc[0][0]; int ai = 0;
      if (acc[0][1] > m) { m = acc[0][1]; ai = 1; }
      if (acc[1][0] > m) { m = acc[1][0]; ai = 2; }
      if (acc[1][1] > m) { m = acc[1][1]; ai = 3; }
      m += sm.wc[75 + c];
      sm.a1[s * A1_STRIDE + c * NPOOL + p] = fmaxf(m, 0.f);
      sm.arg[s * FC1_IN + c * NPOOL + p] = (unsigned char)ai;
    }
  }
}

// ---- tensor-core helpers for the three fc1-sized GEMMs (64 x 432 x <=8 samples) -----------------------------
// The 3xTF32 mma.sync helpers (common.cuh) keep fp32-level accuracy.  A warpgroup-wide wgmma tile does not fit here:
// the split needs hi and lo copies of the 110 KB weight tile in shared memory, and a 64 x 8 output tile would leave
// most of it idle — these GEMMs are latency-, not throughput-bound.

// fc1 pre-activation partials: hpart[kg][s][j] = sum_{k in group kg} W1[j][k] a1[s][k]
// warp w: rows j0 = 16 (w & 3), k-group kg = w >> 2 (9 k-steps of 8)
template <int SPB, int NT>
__device__ __forceinline__ void fc1_forward(Smem<SPB, NT>& sm, int tid) {
  static_assert(NT == 768, "24 warps = 4 row tiles x 6 k-groups");
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int j0 = 16 * (warp & 3), kg = warp >> 2;
  float c[4] = {0.f, 0.f, 0.f, 0.f};
  const float* wa = sm.w1 + (j0 + g) * W1_STRIDE + t;
  const float* xb = sm.a1 + g * A1_STRIDE + t;
#pragma unroll 3
  for (int i = 0; i < 9; ++i) {
    const int k0 = (kg * 9 + i) * 8;
    const FragA a = make_frag_a(wa[k0], wa[8 * W1_STRIDE + k0], wa[k0 + 4], wa[8 * W1_STRIDE + k0 + 4]);
    const FragB b = make_frag_b(xb[k0], xb[k0 + 4]);
    mma3(c, a, b);
  }
  float* hp = sm.hpart + (kg * 8) * HID;
  hp[(2 * t) * HID + j0 + g] = c[0];
  hp[(2 * t + 1) * HID + j0 + g] = c[1];
  hp[(2 * t) * HID + j0 + g + 8] = c[2];
  hp[(2 * t + 1) * HID + j0 + g + 8] = c[3];
}

// stage fc1 weights with the TMA engine (one bulk copy per 1728-byte row into the padded smem rows,
// completion tracked by an mbarrier transaction count) and the small tensors with L2 loads
template <int SPB, int NT>
__device__ __forceinline__ void stage_params(Smem<SPB, NT>& sm, const Args& a, const float* th, int tid) {
  // warp 1 drives the TMA engine (each lane queues two row copies) and warps 2+ fetch the small tensors, so
  // warp 0 is free to run the sampler chain (draw counter -> permutation -> label) that gates the image loads
  const float* w1g = th + a.off_w1;
  if ((tid >> 5) == 1) {
    const int lane = tid & 31;
    if (lane == 0) {
      mbarrier_init(&sm.w1_bar, 1);
      mbarrier_expect_tx(&sm.w1_bar, HID * FC1_IN * 4);
    }
    __syncwarp();
    for (int j = lane; j < HID; j += 32) tma_bulk_g2s(sm.w1 + j * W1_STRIDE, w1g + j * FC1_IN, FC1_IN * 4, &sm.w1_bar);
  }
  if (tid >= 64) {
    const int t2 = tid - 64;
    if (t2 < 75) sm.wc[t2] = __ldcg(th + a.off_wc + t2);
    else if (t2 < 78) sm.wc[t2] = __ldcg(th + a.off_bc + (t2 - 75));
    else if (t2 >= 96 && t2 < 96 + HID) sm.b1[t2 - 96] = __ldcg(th + a.off_b1 + (t2 - 96));
    else if (t2 >= 160 && t2 < 160 + NCLS) sm.b2[t2 - 160] = __ldcg(th + a.off_b2 + (t2 - 160));
    for (int o = t2; o < NCLS * HID; o += NT - 64) sm.w2[o] = __ldcg(th + a.off_w2 + o);
  }
}

// where the minibatch of draw `call` of node l lives
struct BatchGeom { uint32_t bs, start, key, m; int shard_off; float inv_bs; int call; };
template <bool TRAIN>
__device__ __forceinline__ BatchGeom batch_geom(const Args& a, int l, int call) {
  BatchGeom g{0, 0, 0, 0, 0, 1.f, call};
  if (TRAIN) {
    if (a.direct) {
      g.bs = a.direct_bs != nullptr ? (uint32_t)a.direct_bs[l] : (uint32_t)a.batch;
    } else {
      g.m = (uint32_t)a.shard_len[l];
      g.shard_off = a.shard_off[l];
      const BatchLoc loc = locate_batch((uint32_t)call, g.m, (uint32_t)a.batch);
      g.bs = loc.size; g.start = loc.start;
      g.key = mix_key((uint32_t)a.seed, (uint32_t)(a.node0 + l), loc.epoch);
    }
    g.inv_bs = 1.f / (float)(g.bs ? g.bs : 1);
  }
  return g;
}

// optional %globaltimer stamps of the phase boundaries (a.prof, scripts/profile_round_phases.py)
__device__ __forceinline__ void phase_stamp(long long* prof, int idx, int tid) {
  if (prof != nullptr && tid == 0) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    prof[idx] = t;
  }
}

// ---- data half of a step: which samples, then their pixels into the even/odd smem planes --------------------
// Reads only the dataset and the sampler state, never parameters.  `select_samples` returns the label (load in
// flight) for threads < SPB; the caller stores it with `commit_labels` once the images are committed.
template <int SPB, int NT, bool TRAIN>
__device__ __forceinline__ int select_samples(Smem<SPB, NT>& sm, const Args& a, int l, int slice, int chunk,
                                              const BatchGeom& bg, int tid) {
  int lab = 0;   // label load stays in flight across the barrier; it is only needed by the loss
  if (tid < SPB) {
    int idx = 0; float ok = 0.f;
    if (TRAIN) {
      const uint32_t t = slice * SPB + tid;
      if (t < bg.bs) {
        ok = 1.f;
        idx = a.direct ? (int)(l * a.batch + t) : bg.shard_off + (int)feistel_permute(bg.start + t, bg.m, bg.key);
      }
    } else {
      const int t = chunk * SPB + tid;
      if (t < a.n_val) { ok = 1.f; idx = t; }
    }
    sm.sidx[tid] = idx;
    sm.valid[tid] = ok;
    if (ok != 0.f) lab = (int)a.y[idx];
  }
  __syncthreads();
  return lab;
}
template <int SPB, int NT, bool TRAIN>
__device__ __forceinline__ void load_chunk(Smem<SPB, NT>& sm, const Args& a, int l, int slice, int chunk,
                                           const BatchGeom& bg, int tid) {
  const int lab = select_samples<SPB, NT, TRAIN>(sm, a, l, slice, chunk, bg, tid);
  ImgRegs<SPB, NT> r;
  issue_image_loads<SPB, NT>(sm, a, tid, r);
  commit_images<SPB, NT>(sm, a, tid, r);
  if (tid < SPB) sm.label[tid] = lab;
}

// ---- compute half: forward, loss, backward of the SPB samples staged by load_chunk -----------------------------
// Training writes the slice's partial gradient row and loss.
template <int SPB, int NT, bool TRAIN>
__device__ __forceinline__ void compute_chunk(Smem<SPB, NT>& sm, const Args& a, int l, int slice, int S,
                                              const BatchGeom& bg, int tid, long long* prof = nullptr) {
  const float inv_bs = bg.inv_bs;
    if (SPB < 8) {   // sample padding of the MMA operands (never written afterwards)
      for (int o = tid; o < (8 - SPB) * A1_STRIDE; o += NT) sm.a1[SPB * A1_STRIDE + o] = 0.f;
      for (int o = tid; o < HID * 8; o += NT) if ((o & 7) >= SPB) sm.dhT[o] = 0.f;
    }
    __syncthreads();   // images + staged small tensors visible
    phase_stamp(prof, 1, tid);
    conv_relu_pool<SPB, NT>(sm, tid);
    mbarrier_wait_parity(&sm.w1_bar, 0);   // fc1 weights have landed (no-op after the first chunk)
    __syncthreads();
    phase_stamp(prof, 2, tid);

    // ---- fc1 -------------------------------------------------------------------------------
    fc1_forward<SPB, NT>(sm, tid);
    __syncthreads();
    phase_stamp(prof, 3, tid);
    for (int o = tid; o < SPB * HID; o += NT) {
      const int s = o >> 6, j = o & 63;
      float v = sm.b1[j];
#pragma unroll
      for (int kg = 0; kg < KGROUPS; ++kg) v += sm.hpart[(kg * 8 + s) * HID + j];
      sm.h[o] = fmaxf(v, 0.f);
    }
    __syncthreads();
    phase_stamp(prof, 4, tid);

    // ---- fc2 + log-softmax + NLL -----------------------------------------------------------
    {
      // 8 lanes per logit, each over 8 hidden units, then a 3-step shuffle tree (a single thread per logit
      // would be a 64-deep dependent FMA chain)
      const int o = tid >> 3, part = tid & 7;
      const bool live = o < SPB * NCLS;
      const int s = live ? o / NCLS : 0, c = live ? o - s * NCLS : 0;
      float v = 0.f;
      if (live) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = part * 8 + jj;
          v = fmaf(sm.h[s * HID + j], sm.w2[c * HID + j], v);
        }
      }
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      if (live && part == 0) sm.z[s * 16 + c] = v + sm.b2[c];
    }
    __syncthreads();
    phase_stamp(prof, 5, tid);
    if (tid < SPB) {
      const int s = tid;
      float mx = sm.z[s * 16];
      int am = 0;
#pragma unroll
      for (int c = 1; c < NCLS; ++c) if (sm.z[s * 16 + c] > mx) { mx = sm.z[s * 16 + c]; am = c; }
      float se = 0.f;
#pragma unroll
      for (int c = 0; c < NCLS; ++c) se += __expf(sm.z[s * 16 + c] - mx);
      const float lse = mx + __logf(se);
      const int y = sm.label[s];
      const float ok = sm.valid[s];
      const float loss = ok * (lse - sm.z[s * 16 + y]);
      if (TRAIN) {
#pragma unroll
        for (int c = 0; c < NCLS; ++c)
          sm.dz[s * 16 + c] = ok * inv_bs * (__expf(sm.z[s * 16 + c] - lse) - (c == y ? 1.f : 0.f));
        sm.red[s] = loss;
      } else if (ok != 0.f) {
        const size_t o = (size_t)l * a.n_val + sm.sidx[s];
        a.val_loss[o] = loss;
        a.val_correct[o] = (unsigned char)(am == y);
      }
    }
    __syncthreads();
    phase_stamp(prof, 6, tid);
    if (!TRAIN) return;

    float* gp = a.grad_part + ((size_t)l * S + slice) * a.n_pad;
    if (tid == 0) {
      float tot = 0.f;
#pragma unroll
      for (int s = 0; s < SPB; ++s) tot += sm.red[s];
      a.loss_part[l * S + slice] = tot * inv_bs;
      if (a.loss_mirror != nullptr) a.loss_mirror[l * S + slice] = tot * inv_bs;   // zero-copy store to pinned host memory
    }
    // ---- fc2 grads, dh ----------------------------------------------------------------------
    for (int o = tid; o < NCLS * HID; o += NT) {
      const int c = o >> 6, j = o & 63;
      float v = 0.f;
#pragma unroll
      for (int s = 0; s < SPB; ++s) v = fmaf(sm.dz[s * 16 + c], sm.h[s * HID + j], v);
      gp[a.off_w2 + o] = v;
    }
    if (tid < NCLS) {
      float v = 0.f;
#pragma unroll
      for (int s = 0; s < SPB; ++s) v += sm.dz[s * 16 + tid];
      gp[a.off_b2 + tid] = v;
    }
    for (int o = tid; o < SPB * HID; o += NT) {
      const int s = o >> 6, j = o & 63;
      float v = 0.f;
#pragma unroll
      for (int c = 0; c < NCLS; ++c) v = fmaf(sm.dz[s * 16 + c], sm.w2[c * HID + j], v);
      v = sm.h[o] > 0.f ? v : 0.f;
      sm.dh[o] = v;
      sm.dhT[j * 8 + s] = v;
    }
    __syncthreads();
    phase_stamp(prof, 7, tid);
    if (tid < HID) {
      float v = 0.f;
#pragma unroll
      for (int s = 0; s < SPB; ++s) v += sm.dh[s * HID + tid];
      gp[a.off_b1 + tid] = v;
    }
    {
      const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
      // ---- da1[s][k] = relu'(a1) * sum_j dh[s][j] W1[j][k]: out tile [16 k][8 s], A = W1^T, B = dh^T ---------
      for (int mt = warp; mt < FC1_IN / 16; mt += NT / 32) {
        const int k0 = 16 * mt;
        float c[4] = {0.f, 0.f, 0.f, 0.f};
        const float* wa = sm.w1 + t * W1_STRIDE + k0 + g;
        const float* db = sm.dhT + t * 8 + g;
#pragma unroll 4
        for (int js = 0; js < HID / 8; ++js) {
          const int j0 = 8 * js;
          const FragA af = make_frag_a(wa[j0 * W1_STRIDE], wa[j0 * W1_STRIDE + 8], wa[(j0 + 4) * W1_STRIDE],
                                       wa[(j0 + 4) * W1_STRIDE + 8]);
          const FragB bf = make_frag_b(db[j0 * 8], db[(j0 + 4) * 8]);
          mma3(c, af, bf);
        }
        const int s0 = 2 * t, ka = k0 + g, kb = k0 + g + 8;
        if (s0 < SPB) {
          sm.da1[s0 * FC1_IN + ka] = sm.a1[s0 * A1_STRIDE + ka] > 0.f ? c[0] : 0.f;
          sm.da1[s0 * FC1_IN + kb] = sm.a1[s0 * A1_STRIDE + kb] > 0.f ? c[2] : 0.f;
        }
        if (s0 + 1 < SPB) {
          sm.da1[(s0 + 1) * FC1_IN + ka] = sm.a1[(s0 + 1) * A1_STRIDE + ka] > 0.f ? c[1] : 0.f;
          sm.da1[(s0 + 1) * FC1_IN + kb] = sm.a1[(s0 + 1) * A1_STRIDE + kb] > 0.f ? c[3] : 0.f;
        }
      }
      // ---- dW1[j][k] = sum_s dh[s][j] a1[s][k]: one k-step (8 samples); warp = 16 rows x 9 column tiles; the C
      //      fragments go straight to global memory (every store instruction fills eight whole 32-byte sectors)
      {
        const int j0 = 16 * (warp & 3), ng = warp >> 2;
        const float* da = sm.dhT + (j0 + g) * 8 + t;
        const FragA af = make_frag_a(da[0], da[64], da[4], da[68]);
        const float* xb = sm.a1 + t * A1_STRIDE + g;
        float* out = gp + a.off_w1 + (j0 + g) * FC1_IN + 2 * t;
#pragma unroll 3
        for (int i = 0; i < 9; ++i) {
          const int k0 = (ng * 9 + i) * 8;
          const FragB bf = make_frag_b(xb[k0], xb[4 * A1_STRIDE + k0]);
          float c[4] = {0.f, 0.f, 0.f, 0.f};
          mma3(c, af, bf);
          *reinterpret_cast<float2*>(out + k0) = make_float2(c[0], c[1]);
          *reinterpret_cast<float2*>(out + 8 * FC1_IN + k0) = make_float2(c[2], c[3]);
        }
      }
    }
    __syncthreads();   // da1 complete; every read of the staged W1 is done: its smem becomes scratch
    phase_stamp(prof, 8, tid);
    // ---- conv grads: each pooled cell routes da1 to its argmax conv position ------------------
    // 3 groups of 256 threads, one per channel; partial sums are transposed through smem
    // (scratch = the dead W1 region) and reduced by warps — no 26x5 shuffle trees.
    float cacc[26];
#pragma unroll
    for (int i = 0; i < 26; ++i) cacc[i] = 0.f;
    const int cg = tid / CGROUP, ct = tid - cg * CGROUP;
    if (cg < F) {
      for (int it = ct; it < SPB * NPOOL; it += CGROUP) {
        const int s = it / NPOOL, p = it - s * NPOOL;
        const float g = sm.da1[s * FC1_IN + cg * NPOOL + p];
        if (g != 0.f) {
          const int ai = sm.arg[s * FC1_IN + cg * NPOOL + p];
          const int py = p / PHW, pxx = p - py * PHW;
          // window origin (2 py + ai/2, 2 pxx + ai%2): column parity decides which plane serves the even / odd
          // taps, so two base pointers turn every tap into one immediate-offset LDS
          const int par = ai & 1, base = s * XPLANE + (2 * py + (ai >> 1)) * XROW + pxx;
          const float* pA = (par ? sm.xo : sm.xe) + base;        // taps kx = 0, 2, 4
          const float* pB = (par ? sm.xe + 1 : sm.xo) + base;    // taps kx = 1, 3
#pragma unroll
          for (int ky = 0; ky < KS; ++ky)
#pragma unroll
            for (int kx = 0; kx < KS; ++kx)
              cacc[ky * 5 + kx] = fmaf(g, ((kx & 1) ? pB : pA)[ky * XROW + (kx >> 1)], cacc[ky * 5 + kx]);
          cacc[25] += g;
        }
      }
    }
    float* scratch = sm.w1;   // [78][CGROUP]
    if (cg < F) {
#pragma unroll
      for (int i = 0; i < 26; ++i) scratch[(cg * 26 + i) * CGROUP + ct] = cacc[i];
    }
    __syncthreads();
    phase_stamp(prof, 9, tid);
    {
      const int warp = tid >> 5, lane = tid & 31;
      for (int o = warp; o < 78; o += NT / 32) {
        float v = 0.f;
#pragma unroll
        for (int q = 0; q < CGROUP / 32; ++q) v += scratch[o * CGROUP + lane + 32 * q];
        v = warp_sum(v);
        if (lane == 0) {
          const int c = o / 26, i = o - c * 26;
          gp[(i < 25) ? a.off_wc + c * 25 + i : a.off_bc + c] = v;
        }
      }
    }
}

}  // namespace mnist
}  // namespace nndt

namespace nndt {
namespace mnist {
template <int SPB, int NT, bool TRAIN>
__device__ __forceinline__ void process_chunk(Smem<SPB, NT>& sm, const Args& a, int l, int slice, int S, int chunk,
                                              const BatchGeom& bg, int tid) {
  load_chunk<SPB, NT, TRAIN>(sm, a, l, slice, chunk, bg, tid);
  compute_chunk<SPB, NT, TRAIN>(sm, a, l, slice, S, bg, tid);
}
}  // namespace mnist
}  // namespace nndt
