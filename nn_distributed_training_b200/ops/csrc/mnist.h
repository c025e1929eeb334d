// Launch interface of the fused MNIST conv-net kernels (mnist.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nndt {
namespace mnist {

struct Args {
  // parameters: row l of theta [L, n_pad]; slot offsets from FlatLayout
  const float* theta;
  int n_pad, L;
  int off_wc, off_bc, off_w1, off_b1, off_w2, off_b2;
  // data (uint8 pixels + (mean, 1/std), or float32 already normalised), int64 labels
  const void* x;
  const int64_t* y;
  int x_is_u8;
  float mean, inv_std;
  // sampling: direct==1 -> rows [l*batch + t]; else stateless permutation of shard l
  int direct, batch, seed, node0;
  const int* direct_bs;   // [L] valid rows per node when direct (nullptr: all `batch`)
  const int* shard_off;   // [L]
  const int* shard_len;   // [L]
  int* calls;             // [L] draw counter per node (device); the training kernel advances it itself
  unsigned int* arrive;   // [L] CTA arrival counters used to advance `calls` exactly once per launch
  int tune;               // bit 0: sampler chain + row gather issued before the PDL wait
  long long* prof;        // optional [L*S, 64] %globaltimer stamps (scripts/profile_round_phases.py); nullptr = off
  // training outputs
  float* grad_part;       // [L, S, n_pad]
  float* loss_part;       // [L, S]
  float* loss_mirror;     // [L, S] optional second destination in pinned host memory (device-initiated D2H of the result)
  // evaluation
  int n_val;
  float* val_loss;              // [L, n_val]
  unsigned char* val_correct;   // [L, n_val]
};

// Device-initiated host->device staging: the GPU pulls the next round's minibatch rows straight out of the
// *pinned host* dataset (UVA pointer, PCIe reads) with the stateless sampler and writes them to a device
// staging set.  No CPU work per round.
struct GatherArgs {
  const unsigned char* x_host;   // pinned host rows [M_total, row_bytes]
  const int64_t* y_host;         // pinned host labels [M_total]
  int row_bytes;
  unsigned char* x_stage;        // device [P, L, B, row_bytes]
  int64_t* y_stage;              // device [P, L, B]
  int* bs_stage;                 // device [P, L]
  int P, L, batch, seed, node0;
  const int* shard_off; const int* shard_len;
  const int* calls0;             // [L] draw counters at round 0 of the stream
  int* stage_round;              // [1] device counter of staged rounds (advanced by this kernel)
  unsigned int* done_ctr;        // [1]
  int max_blocks;                // grid cap: the staging blocks must leave one SM per concurrent training CTA
};
// Generic CUDA-core conv net (mnist_generic.cu): any (num_filters <= 8, kernel_size in {3,5}, linear_width <= 128), fp32 or
// fp64.  With dtype64 the Args pointers theta / grad_part / val_loss address doubles (loss_part stays float).
struct GenericShape { int F, KS, LW, dtype64; double mean, inv_std; };   // mean / inv_std in full precision for the fp64 arm
size_t generic_smem_bytes(const GenericShape& gs, int dtype64, int spb);
int generic_eval_spb(const GenericShape& gs);   // samples per CTA of launch_generic_eval: 8, or 4 past 160 KB of smem
cudaError_t launch_generic_train(const Args& a, const GenericShape& gs, int spb, int S, cudaStream_t st);
cudaError_t launch_generic_eval(const Args& a, const GenericShape& gs, int ctas_per_node, cudaStream_t st);
// Tensor-core training kernel of the paper shape (mnist_tc.cu): K-split over a 6-CTA cluster per node, batch <= 64,
// ONE gradient row per node (S = 1).  `w1_map128` = the 128-byte CUtensorMap written by make_w1_tensor_map.
cudaError_t make_w1_tensor_map(const float* theta, int n_pad, int L, int off_w1, void* out_map128);
cudaError_t launch_train_tc(const Args& a, const void* w1_map128, int nsplit, cudaStream_t st);
int tc_max_active_clusters();
// float64 K-split cluster kernel of the paper shape on the FP64 tensor cores (mnist_cl64.cu): nsplit clusters of
// cl64_cluster_ctas() CTAs per node, one gradient row per cluster; Args pointers address doubles
cudaError_t launch_train_cl64(const Args& a, const GenericShape& gs, int nsplit, cudaStream_t st);
int cl64_max_active_clusters(int nsplit);
int cl64_cluster_ctas();
cudaError_t launch_gather(const GatherArgs& a, cudaStream_t st);
cudaError_t launch_train(const Args& a, int spb, int S, cudaStream_t st);
cudaError_t launch_eval(const Args& a, int ctas_per_node, cudaStream_t st);
cudaError_t launch_batch_indices(int m, int B, int call, int seed, int node, int* out, int* out_size, cudaStream_t st);

}  // namespace mnist
}  // namespace nndt
