// Launch interface of the PPO update kernels (ppo_update.cu): advantages and every node's actor and critic gradients.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nndt {
namespace ppo {

constexpr int kMaxNodes = 8, kMaxLayers = 5, kMaxWidth = 64, kActDim = 5;
constexpr int kActor = 0, kCritic = 1;

// One ReLU MLP with biases: nn.Linear's row-major [dims[l+1], dims[l]] weight W[l] and bias b[l], read in place, and
// the tensors the gradient kernel writes their gradients to (same shapes; only grads() needs them).
struct Net {
  const void* W[kMaxLayers];
  const void* b[kMaxLayers];
  void* gW[kMaxLayers];
  void* gb[kMaxLayers];
};

struct Args {
  int dtype64;
  int N, R;                        // nodes, samples per node
  int nl[2];                       // linear layers of the actor / critic (actor: 0 for advantages())
  int dims[2][kMaxLayers + 1];     // actor [obs_dim, .., 5], critic [obs_dim, .., 1]
  Net net[kMaxNodes][2];
  // Batch, row r of node i at [i * R + r]: obs [N, R, obs_dim], acts [N, R, 5], old_lp / rtgs / adv [N, R]
  const void* obs;
  const void* acts;
  const void* old_lp;
  const void* rtgs;
  void* adv;                       // input of grads(), output of advantages()
  double clip, cov_var, lp_const;  // lp = -0.5 |act - mean|^2 / cov_var - lp_const
  void* losses;                    // [N, 2]: actor, critic loss
  int* nonfinite;                  // set to 1 if an actor mean is not finite; never cleared
  // GAE(lambda) of advantages() (gae != 0): per-cycle rewards rews [N, R] in the rollout's row order
  // r = (blk * T + c) * E + e, with T * E dividing R; the lambda-returns A + V go to returns [N, R], raw A to adv
  // before the normalisation.  gae == 0: none of these is read, and adv = normalised (rtgs - V).
  int gae, T, E;
  double gamma, lam;
  const void* rews;
  void* returns;
  void* values;                    // optional [N, R]: the critic's V
};

// Rows per tile, chunks per node (CTAs per network), dynamic shared memory, accumulator slot size (doubles) and
// workspace of one launch.  The plan depends on the device (SM count, occupancy) and the shapes, never on the data.
struct Plan {
  int tm, chunks;
  size_t smem, gmax, work_bytes;
  cudaError_t err;   // cudaSuccess, or why the kernels cannot launch this configuration
};

// nullptr if the kernels support a, otherwise the reason; without the actor (advantages) only the critic is described
// (nl[kActor] may be 0) and no gradient outputs are needed.
const char* check(const Args& a, bool with_actor);
// Cached per (device, dtype, pass, shapes, N, R): the device queries run once, not once per primal step.
Plan plan(const Args& a, bool backward);
// grads(): losses and every gradient with p = plan(a, true); `work` holds p.work_bytes.
cudaError_t grads(const Args& a, const Plan& p, void* work, cudaStream_t st);
// advantages(): adv = normalised (rtgs - critic(obs)) per node; with a.gae, adv = normalised GAE(lambda) advantages
// and returns = their lambda-returns.
cudaError_t advantages(const Args& a, cudaStream_t st);

}  // namespace ppo
}  // namespace nndt
