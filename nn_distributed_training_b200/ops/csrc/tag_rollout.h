// Launch interface of the fused multi-agent PPO rollout on the predator-prey environment (tag_rollout.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nndt {
namespace tag {

constexpr int kMaxAgents = 8, kMaxPred = kMaxAgents - 1, kMaxObst = 8;
constexpr int kMaxLayers = 5, kMaxWidth = 64, kActDim = 5;

struct Args {
  int dtype64;
  // Actors: n_actor distinct ReLU MLPs [dims[0], .., dims[nl] = 5]; predator i runs actor actor_of[i].  W[a][l] is
  // nn.Linear's [dims[l+1], dims[l]] row-major weight, b[a][l] its bias, both read in place.
  int n_actor, nl;
  int actor_of[kMaxPred];
  int dims[kMaxLayers + 1];
  const void* W[kMaxPred][kMaxLayers];
  const void* b[kMaxPred][kMaxLayers];
  // Environment: N predators (agents 0..N-1), n_good prey, A = N + n_good agents, n_obst immovable obstacles.
  int N, n_good, A, n_obst;
  const void* size;        // [A]
  const void* accel;       // [A]
  const void* max_speed;   // [A]
  const void* obst;        // [n_obst, 2]
  // Rollout: n_ep episodes of E worlds, T cycles each; world g = ep * E + e starts at pos0[g] with zero velocity.
  int E, n_ep, T;
  const void* pos0;        // [n_ep, E, A, 2]
  double gamma, cov_var, noise_std, lp_const;   // act = mean + noise_std * eps; lp = -0.5 |act-mean|^2 / cov_var - lp_const
  uint64_t key;
  uint32_t index;
  // Outputs, row r = (ep * T + c) * E + e.
  void* obs;               // [N, R, dims[0]]
  void* acts;              // [N, R, 5]
  void* log_probs;         // [N, R]
  void* rtgs;              // [N, R]
  void* ep_returns;        // [n_ep * E]
  void* final_pos;         // [n_ep, E, A, 2]
  void* final_vel;         // [n_ep, E, A, 2]
  void* eps;               // optional [N, R, 5]
  void* pos_trace;         // optional [n_ep, T, E, A, 2], positions after each cycle
  void* rews;              // optional [N, R], the shared predator reward of each cycle (before the rewards-to-go)
};

// Worlds per CTA, whether the actors are staged in shared memory, worlds per register block (the kernel's RW: 4 when
// wpb is a multiple of 4, else 1) and shared memory per CTA for this launch.
struct Plan {
  int wpb, stage, rw;
  size_t smem;
};

const char* check(const Args& a);      // nullptr if the kernel supports a, otherwise the reason
Plan plan(const Args& a);
cudaError_t launch(const Args& a, cudaStream_t st);

}  // namespace tag
}  // namespace nndt
