// Shared device helpers for the sm_90a kernels of nn_distributed_training_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdlib>
#include <utility>

#define NNDT_DEVINL __device__ __forceinline__

namespace nndt {

constexpr int kWarp = 32;

NNDT_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
NNDT_DEVINL double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- system-scope flags for cross-GPU producer/consumer sync -----------------
// A rank publishes round k by (1) writing its rows, (2) __threadfence_system(),
// (3) st.release.sys of k into the *reader's* flag slot (remote store over NVLink),
// so readers spin on local memory only.
NNDT_DEVINL void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
NNDT_DEVINL int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
NNDT_DEVINL int ld_relaxed_sys(const int* p) {
  int v;
  asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// streaming 128-bit load that bypasses L1 allocation (peer / read-once data)
NNDT_DEVINL float4 ld_stream_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// ---- programmatic dependent launch (PDL) -------------------------------------------------------
// Kernels of a round are launched with cudaLaunchAttributeProgrammaticStreamSerialization: a kernel may
// start while its predecessor drains.  Convention in this repo: every kernel executes pdl_wait() before it
// touches anything the *immediately preceding* kernel wrote, and only then pdl_launch_dependents() — so when
// a kernel's pre-wait prologue runs, everything two or more kernels back is complete and visible.
NNDT_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
NNDT_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  static const bool no_pdl = getenv("NNDT_NO_PDL") != nullptr;   // debugging / A-B switch
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
// launch_pdl for a kernel run as thread-block clusters of `cluster_x` CTAs along x: the PDL and cluster-dimension
// attributes go through cudaLaunchKernelEx together
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, int cluster_x,
                                      cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  static const bool no_pdl = getenv("NNDT_NO_PDL") != nullptr;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster_x; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = no_pdl ? 1 : 2;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ---- TMA bulk copy (cp.async.bulk, SASS: UBLKCP) + mbarrier transaction tracking ---------------------
NNDT_DEVINL uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
NNDT_DEVINL void mbarrier_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
NNDT_DEVINL void mbarrier_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(bytes) : "memory");
}
// one thread: copy `bytes` (multiple of 16, 16 B aligned both sides) global -> shared, completing on `bar`
NNDT_DEVINL void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_addr_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_addr_u32(bar))
               : "memory");
}
NNDT_DEVINL void mbarrier_wait_parity(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_addr_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}

// ---- thread-block clusters: barrier, rank, and fp64 distributed-shared-memory access -----------------------------
NNDT_DEVINL void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
NNDT_DEVINL uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
NNDT_DEVINL uint32_t map_to(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(rank));
  return r;
}
NNDT_DEVINL double ld_dsmem(uint32_t a) { double v; asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory"); return v; }
NNDT_DEVINL void st_dsmem(uint32_t a, double v) { asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
NNDT_DEVINL uint32_t ld_dsmem_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
NNDT_DEVINL unsigned long long ld_dsmem_u64(uint32_t a) {
  unsigned long long v;
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
  return v;
}

// ---- cluster pushes: a producer stores into a peer's shared memory and the bytes complete a transaction count on the
//      peer's mbarrier (release at cluster scope); the consumer waits on its own mbarrier for just those bytes.  Both
//      addresses come from map_to() for the consumer's rank ------------------------------------------------------------
NNDT_DEVINL void st_async(uint32_t a, double v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.f64 [%0], %1, [%2];" ::"r"(a), "d"(v), "r"(bar) : "memory");
}
NNDT_DEVINL void st_async(uint32_t a, double v0, double v1, uint32_t bar) {   // 16-byte aligned pair
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f64 [%0], {%1, %2}, [%3];" ::"r"(a), "d"(v0), "d"(v1), "r"(bar)
               : "memory");
}
// the relaxed half of a split cluster barrier: the arrive after this CTA's mbarrier inits, the wait before its first push
NNDT_DEVINL void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
NNDT_DEVINL void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// mbarrier_wait_parity with acquire at cluster scope: the bytes were written by peers' st_async
NNDT_DEVINL void mbarrier_wait_parity_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_addr_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}

// ---- FP64 tensor-core tiles (DMMA) ------------------------------------------------------------------------------
// m16n8k4 fragments (g = lane >> 2, t = lane & 3): A a0 (g, t), a1 (g + 8, t); B b0 (t, g);
// C c0 (g, 2t), c1 (g, 2t + 1), c2 (g + 8, 2t), c3 (g + 8, 2t + 1).
NNDT_DEVINL void dmma(double (&c)[4], double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a0), "d"(a1), "d"(b));
}

// c[j] += sum_k A(m0 + ., k) B(k, n0 + 8 j + .) over k < K (a multiple of 4)
template <int NJ, class FA, class FB>
NNDT_DEVINL void gemm(double (&c)[NJ][4], int m0, int n0, int K, int lane, FA A, FB B) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll 4
  for (int k0 = 0; k0 < K; k0 += 4) {
    const int k = k0 + t;
    const double a0 = A(m0 + g, k), a1 = A(m0 + g + 8, k);
#pragma unroll
    for (int j = 0; j < NJ; ++j) dmma(c[j], a0, a1, B(k, n0 + 8 * j + g));
  }
}

template <int NJ>
NNDT_DEVINL void zero(double (&c)[NJ][4]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.0;
}
// row / column of accumulator element i of the 16 x 8 tile at (m0, n0)
NNDT_DEVINL int frow(int m0, int lane, int i) { return m0 + (lane >> 2) + 8 * (i >> 1); }
NNDT_DEVINL int fcol(int n0, int lane, int i) { return n0 + 2 * (lane & 3) + (i & 1); }

// operand readers: at(s, ld)(i, j) = s[i][j], at_t(s, ld)(i, j) = s[j][i] of a row-major array with row stride ld
template <class T> NNDT_DEVINL auto at(const T* s, int ld) { return [s, ld](int i, int j) { return s[i * ld + j]; }; }
template <class T> NNDT_DEVINL auto at_t(const T* s, int ld) { return [s, ld](int i, int j) { return s[j * ld + i]; }; }

// ---- FP32 on TF32 tensor cores with the 3xTF32 split ----------------------------------------------------------
// mma.sync m16n8k8 TF32 with x = hi + lo (both TF32) and a.b ~ a_lo.b_hi + a_hi.b_lo + a_hi.b_hi, which keeps
// fp32-level accuracy: the framework's contract is fp32 training, not TF32.
// Fragment coordinates (g = lane >> 2, t = lane & 3):
//   A (16x8, row major): a0 (g, t) a1 (g+8, t) a2 (g, t+4) a3 (g+8, t+4)
//   B (8x8, col major) : b0 (k=t, n=g) b1 (k=t+4, n=g)
//   C (16x8)           : c0 (g, 2t) c1 (g, 2t+1) c2 (g+8, 2t) c3 (g+8, 2t+1)   (as the DMMA tile)
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
struct FragA { uint32_t hi[4], lo[4]; };
struct FragB { uint32_t hi[2], lo[2]; };
__device__ __forceinline__ FragA make_frag_a(float a0, float a1, float a2, float a3) {
  FragA f;
  split_tf32(a0, f.hi[0], f.lo[0]); split_tf32(a1, f.hi[1], f.lo[1]);
  split_tf32(a2, f.hi[2], f.lo[2]); split_tf32(a3, f.hi[3], f.lo[3]);
  return f;
}
__device__ __forceinline__ FragB make_frag_b(float b0, float b1) {
  FragB f;
  split_tf32(b0, f.hi[0], f.lo[0]); split_tf32(b1, f.hi[1], f.lo[1]);
  return f;
}
__device__ __forceinline__ void mma3(float (&c)[4], const FragA& a, const FragB& b) {
  mma_tf32(c, a.lo, b.hi);   // small terms first
  mma_tf32(c, a.hi, b.lo);
  mma_tf32(c, a.hi, b.hi);
}

// The fp32 counterpart of gemm(): c[j] += sum_k A(m0 + ., k) B(k, n0 + 8 j + .) over k < K (a multiple of 8), 3xTF32
template <int NJ, class FA, class FB>
NNDT_DEVINL void gemm(float (&c)[NJ][4], int m0, int n0, int K, int lane, FA A, FB B) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll 2
  for (int k0 = 0; k0 < K; k0 += 8) {
    const int k = k0 + t;
    const FragA a = make_frag_a(A(m0 + g, k), A(m0 + g + 8, k), A(m0 + g, k + 4), A(m0 + g + 8, k + 4));
#pragma unroll
    for (int j = 0; j < NJ; ++j) mma3(c[j], a, make_frag_b(B(k, n0 + 8 * j + g), B(k + 4, n0 + 8 * j + g)));
  }
}

// cp.async helpers (LDGSTS)
NNDT_DEVINL void cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
NNDT_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
NNDT_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

}  // namespace nndt
