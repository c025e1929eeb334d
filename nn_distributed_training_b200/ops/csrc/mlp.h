// Launch interface of the tensor-core MLP kernels (mlp_tc.cu: bf16, mlp_f64.cu: fp64): networks of the form
//   d_in (<= 4) -> H1 (64|128|256) -> 64 -> 64 -> 64 -> 1
// i.e. the reference's FourierNet [2,256,64,64,64,1] (models/fourier_nn.py:43-59) and ReLU MLPs
// of the same shape family (models/relu_nn.py:4-41).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nndt {
namespace mlp {

enum FirstAct : int { kFirstRelu = 0, kFirstSinRelu = 1 };
enum LastAct : int { kLastNone = 0, kLastSigmoid = 1 };
enum Loss : int { kLossBCE = 0, kLossMSE = 1, kLossL1 = 2 };

struct Args {
  const float* theta;   // [L, n_pad]
  int n_pad, L;
  int off[10];          // slot offsets: W0,b0,W1,b1,W2,b2,W3,b3,W4,b4
  int d_in, h1;
  int first_act, last_act, loss;
  float scale;
  double scale64;       // the SIREN scale in full precision (fp64 kernels)
  // data: x [M, d_in] fp32 (or fp64 converted by the caller), y [M] fp32
  const float* x;
  const float* y;
  // forward-only
  int n_rows;           // rows evaluated per node (same inputs for every node)
  float* out;           // [L, n_rows] network output
  // training (see mlp_tc.cu)
  int direct, batch, seed, node0;
  const int* shard_off; const int* shard_len; const int* calls;
  const int64_t* win_table;  // online sliding-window tables (nullptr: plain epoch sampling)
  float* grad_part;     // [L, S, n_pad]
  float* loss_part;     // [L, S]
  int S;
};

cudaError_t launch_forward(const Args& a, int ctas_per_node, cudaStream_t st);
cudaError_t launch_train(const Args& a, int ctas, cudaStream_t st);

// float64 kernels (mlp_f64.cu): DMMA tiles on 2-CTA clusters.  With them every pointer of Args except the index
// arrays (shard_off, shard_len, calls, win_table) addresses doubles: theta, x, y, out, grad_part and loss_part.
// Widths count clusters: `clusters_per_node` for the forward kernel, `clusters` for the training kernel, whose
// CTA 2 c + r of cluster c owns slot 2 (c - first cluster of the node) + r, so S >= 2 (clusters per node + 1).
cudaError_t launch_forward_f64(const Args& a, int clusters_per_node, cudaStream_t st);
cudaError_t launch_train_f64(const Args& a, int clusters, cudaStream_t st);
int f64_max_active_clusters(int h1);   // co-resident clusters of the training kernel (0: not launchable)

}  // namespace mlp
}  // namespace nndt
