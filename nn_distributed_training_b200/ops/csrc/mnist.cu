// Fused forward+backward (and forward-only evaluation) of the MNIST conv classifier
//   conv 1->3 5x5 -> ReLU -> maxpool2 -> fc 432->64 -> ReLU -> fc 64->10 -> log-softmax -> NLL
// for every graph node hosted by this GPU in ONE launch (reference op chain:
// models/mnist_conv_nn.py:16-25 driven by problems/dist_mnist_problem.py:96-98, where it is
// ~30 eager ATen/cuDNN launches per node and step).  The device code lives in mnist_device.cuh.
//
// Work decomposition: grid = (S batch slices, L nodes); a CTA of 768 threads owns SPB samples of one node, and the
// Python side picks SPB (4..8) so that S x L CTAs fill the SMs in one wave.  The 110 KB fc1 weight matrix is
// staged per CTA by the TMA engine (cp.async.bulk per padded row, mbarrier transaction count) while warp 0 runs
// the stateless Feistel sampler and the row gather, so there is no host work, no index tensor and no H2D copy per
// step; conv+ReLU+pool run out of an even/odd column-split image tile; fc1 / da1 / dW1 are mma.sync 3xTF32
// tensor-core GEMMs (fp32-accurate).  Each CTA writes its slice's partial gradient row; the consensus update
// kernel that follows sums the S partials while applying the optimizer step (no separate reduce launch).
//
// Batch 64 x 28k parameters is far below a large tensor-core tile's break-even (the whole fc1 GEMM is 1.8 MFLOP, and
// the fp32-accurate operand split would need two copies of the weight tile in shared memory) — DESIGN.md §3.1.
#include "mnist_device.cuh"

namespace nndt {
namespace mnist {

template <int SPB, int NT, bool TRAIN>
__global__ void __launch_bounds__(NT, 1) mnist_kernel(const Args a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem<SPB, NT>& sm = *reinterpret_cast<Smem<SPB, NT>*>(smem_raw);
  const int tid = threadIdx.x;
  const int l = blockIdx.y;
  const float* th = a.theta + (size_t)l * a.n_pad;
  if (TRAIN) {
    // The minibatch depends only on the dataset and on this kernel family's own draw counter (last written by the
    // previous forward/backward launch, i.e. at least two launches back and therefore complete), so with
    // tune bit 0 the sampler chain and the HBM row gather are issued BEFORE the programmatic-dependency wait,
    // while the consensus kernel is still producing the parameters; the pixels are converted after the wait,
    // under the shadow of the parameter staging.
    long long* prof = a.prof != nullptr ? a.prof + (l * gridDim.x + blockIdx.x) * 64 : nullptr;
    phase_stamp(prof, 20, tid);
    const bool early = (a.tune & 1) != 0;
    if (!early) {
      pdl_wait();
      pdl_launch_dependents();
      stage_params<SPB, NT>(sm, a, th, tid);    // TMA + small loads fly while the sampler chain runs
    }
    const int call = a.calls != nullptr ? a.calls[l] : 0;
    const BatchGeom bg = batch_geom<true>(a, l, call);
    const int lab = select_samples<SPB, NT, true>(sm, a, l, blockIdx.x, 0, bg, tid);
    phase_stamp(prof, 21, tid);
    ImgRegs<SPB, NT> img;
    issue_image_loads<SPB, NT>(sm, a, tid, img);
    if (tid == 0 && a.calls != nullptr && a.arrive != nullptr) {
      // the last CTA of the node to get here (all have read the counter) advances it
      if (atomicAdd(a.arrive + l, 1u) == gridDim.x - 1) { a.arrive[l] = 0; a.calls[l] = call + 1; }
    }
    if (early) {
      pdl_wait();               // parameters of this step are now final
      pdl_launch_dependents();
      phase_stamp(prof, 22, tid);
      stage_params<SPB, NT>(sm, a, th, tid);
    }
    commit_images<SPB, NT>(sm, a, tid, img);
    if (tid < SPB) sm.label[tid] = lab;
    compute_chunk<SPB, NT, true>(sm, a, l, blockIdx.x, gridDim.x, bg, tid, prof);
    phase_stamp(prof, 23, tid);
  } else {
    pdl_wait();
    pdl_launch_dependents();
    stage_params<SPB, NT>(sm, a, th, tid);
    const BatchGeom bg = batch_geom<false>(a, l, 0);
    const int n_chunks = (a.n_val + SPB - 1) / SPB;
    for (int chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x)
      process_chunk<SPB, NT, false>(sm, a, l, blockIdx.x, gridDim.x, chunk, bg, tid);
  }
}

constexpr int kNT = 768;

template <int SPB, bool TRAIN>
static cudaError_t prepare_once() {
  // opt in to >48 KB dynamic shared memory once per process (not a stream op: legal under capture)
  static cudaError_t st = cudaFuncSetAttribute(mnist_kernel<SPB, kNT, TRAIN>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)sizeof(Smem<SPB, kNT>));
  return st;
}

template <int SPB>
static cudaError_t launch_t(const Args& a, int S, bool train, int eval_ctas, cudaStream_t st) {
  const size_t smem = sizeof(Smem<SPB, kNT>);
  cudaError_t e = train ? prepare_once<SPB, true>() : prepare_once<SPB, false>();
  if (e != cudaSuccess) return e;
  if (train) {
    return launch_pdl(mnist_kernel<SPB, kNT, true>, dim3(S, a.L), dim3(kNT), smem, st, a);
  } else {
    mnist_kernel<SPB, kNT, false><<<dim3(eval_ctas, a.L), kNT, smem, st>>>(a);
  }
  return cudaGetLastError();
}

// ---- device-initiated H2D staging of one round's minibatches (one warp per row) -------------------------
constexpr int kGatherThreads = 512;
__global__ void __launch_bounds__(kGatherThreads) gather_rows_kernel(const GatherArgs a) {
  // few, long-lived blocks: the staging copy must leave the SMs (and their register files) to the training CTAs
  // it overlaps with.  PCIe reads have microseconds of latency, so each warp keeps TWO rows (1.5 KB) in flight.
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int rows = a.P * a.L * a.batch;
  const int r = *a.stage_round;
  const int n16 = a.row_bytes >> 4;
  const int w0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  for (int row0 = w0; row0 < rows; row0 += 2 * nwarps) {
    const uint4* s4[2] = {nullptr, nullptr};
    uint4* d4[2] = {nullptr, nullptr};
    uint4 v[2][2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int row = row0 + u * nwarps;
      v[u][0] = v[u][1] = make_uint4(0, 0, 0, 0);
      if (row >= rows) continue;
      const int t = row % a.batch, l = (row / a.batch) % a.L, p = row / (a.batch * a.L);
      const uint32_t m = (uint32_t)a.shard_len[l];
      const BatchLoc loc = locate_batch((uint32_t)(a.calls0[l] + r * a.P + p), m, (uint32_t)a.batch);
      if (t == 0 && lane == 0) a.bs_stage[p * a.L + l] = (int)loc.size;
      if ((uint32_t)t >= loc.size) continue;
      const uint32_t key = mix_key((uint32_t)a.seed, (uint32_t)(a.node0 + l), loc.epoch);
      const size_t src = (size_t)a.shard_off[l] + feistel_permute(loc.start + t, m, key);
      s4[u] = reinterpret_cast<const uint4*>(a.x_host + src * a.row_bytes);
      d4[u] = reinterpret_cast<uint4*>(a.x_stage + (size_t)row * a.row_bytes);
      if (lane < n16) v[u][0] = s4[u][lane];
      if (lane + 32 < n16) v[u][1] = s4[u][lane + 32];
      if (lane == 0) a.y_stage[row] = a.y_host[src];
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (d4[u] == nullptr) continue;
      if (lane < n16) d4[u][lane] = v[u][0];
      if (lane + 32 < n16) d4[u][lane + 32] = v[u][1];
      for (int i = lane + 64; i < n16; i += 32) d4[u][i] = s4[u][i];
    }
  }
  // last block advances the staged-round counter
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(a.done_ctr, 1u) == gridDim.x - 1;
  __syncthreads();
  if (is_last && threadIdx.x == 0) { *a.done_ctr = 0; *a.stage_round = r + 1; }
}
cudaError_t launch_gather(const GatherArgs& a, cudaStream_t st) {
  const int rows = a.P * a.L * a.batch;
  int blocks = (rows * 32 + kGatherThreads - 1) / kGatherThreads;
  const int cap = a.max_blocks > 0 ? a.max_blocks : 24;
  if (blocks > cap) blocks = cap;
  gather_rows_kernel<<<blocks, kGatherThreads, 0, st>>>(a);
  return cudaGetLastError();
}

// debug/test helper: the sampler's row indices for one draw (mirrors data/sampler.py)
__global__ void batch_indices_kernel(int m, int B, int call, int seed, int node, int* out, int* out_size) {
  const BatchLoc loc = locate_batch((uint32_t)call, (uint32_t)m, (uint32_t)B);
  const uint32_t key = mix_key((uint32_t)seed, (uint32_t)node, loc.epoch);
  for (uint32_t t = threadIdx.x; t < loc.size; t += blockDim.x)
    out[t] = (int)feistel_permute(loc.start + t, (uint32_t)m, key);
  if (threadIdx.x == 0) *out_size = (int)loc.size;
}
cudaError_t launch_batch_indices(int m, int B, int call, int seed, int node, int* out, int* out_size, cudaStream_t st) {
  batch_indices_kernel<<<1, 256, 0, st>>>(m, B, call, seed, node, out, out_size);
  return cudaGetLastError();
}

cudaError_t launch_train(const Args& a, int spb, int S, cudaStream_t st) {
  // samples per CTA: the Python side picks the value that best fills the SMs with L x ceil(batch / spb) CTAs
  switch (spb) {
    case 4: return launch_t<4>(a, S, true, 0, st);
    case 5: return launch_t<5>(a, S, true, 0, st);
    case 6: return launch_t<6>(a, S, true, 0, st);
    case 7: return launch_t<7>(a, S, true, 0, st);
    case 8: return launch_t<8>(a, S, true, 0, st);
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_eval(const Args& a, int ctas_per_node, cudaStream_t st) {
  return launch_t<8>(a, 0, false, ctas_per_node, st);
}

}  // namespace mnist
}  // namespace nndt