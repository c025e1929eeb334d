// Device-side helpers of the consensus kernels (consensus.cu).
#pragma once
#include <curand_philox4x32_x.h>

#include "common.cuh"
#include "consensus.h"

namespace nndt {
namespace consensus {

constexpr int THREADS = 256;
constexpr long long kSpinLimit = 20000000000LL;  // ~10 s at 2 GHz, then flag an error and go on

template <typename T> struct Vec;
template <> struct Vec<float> { using type = float4; static constexpr int N = 4; };
template <> struct Vec<double> { using type = double2; static constexpr int N = 2; };

template <typename T> struct Pack { T v[Vec<T>::N]; };

template <typename T>
NNDT_DEVINL Pack<T> ldv(const T* p) {
  Pack<T> r;
  *reinterpret_cast<typename Vec<T>::type*>(r.v) = *reinterpret_cast<const typename Vec<T>::type*>(p);
  return r;
}
template <typename T>
NNDT_DEVINL void stv(T* p, const Pack<T>& r) {
  *reinterpret_cast<typename Vec<T>::type*>(p) = *reinterpret_cast<const typename Vec<T>::type*>(r.v);
}

template <typename T>
struct RoundInfo { int k, par, gid; };

template <typename T>
NNDT_DEVINL RoundInfo<T> round_info(const Common<T>& c) {
  RoundInfo<T> r;
  r.k = *c.round_ctr;
  r.par = r.k & 1;
  r.gid = c.graph_id[r.k];
  return r;
}

// local node handled by this CTA row: nodes whose neighbors live on other GPUs are launched first, so their NVLink
// pulls run in the shadow of the preceding forward/backward kernel (the update grid only becomes fully resident when
// that kernel drains)
template <typename T>
NNDT_DEVINL int node_of_block(const Common<T>& c) {
  return c.node_order != nullptr ? c.node_order[blockIdx.y] : (int)blockIdx.y;
}

// A kernel that prefetches what the preceding kernel does not write calls this after its first loads and once more
// after its loop: the first call waits for that kernel (griddepcontrol.wait) and lets the next one launch, the others
// do nothing.  The second call covers a thread that got no loop iteration.
NNDT_DEVINL void release_dependents_once(bool& waited) {
  if (!waited) { pdl_wait(); pdl_launch_dependents(); waited = true; }
}

// debug timeline: stamp `which` (0..7) of update launch (round k, primal step) by the first and the last block of the grid
template <typename T>
NNDT_DEVINL void tl_stamp(const Common<T>& c, int k, int step, int which) {
  if (c.timeline == nullptr || threadIdx.x != 0) return;
  const bool first = blockIdx.x == 0 && blockIdx.y == 0, last = blockIdx.x == gridDim.x - 1 && blockIdx.y == gridDim.y - 1;
  if (!first && !last) return;
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  c.timeline[(size_t)((k * 4 + step) & 4095) * 16 + (first ? 0 : 8) + which] = t;
}

// spin until rank r has published round k (the peer stores into our local slot)
template <typename T>
NNDT_DEVINL void wait_rank(const Common<T>& c, int r, int k) {
  const int* f = c.flags + r;
  if (ld_acquire_sys(f) >= k) return;
  if (*reinterpret_cast<volatile int*>(c.err) != 0) return;      // a peer already timed out: do not stack 10 s spins
  const long long t0 = clock64();
  while (ld_acquire_sys(f) < k) {
    if (clock64() - t0 > kSpinLimit) { *c.err = 1; break; }
  }
}

// Round-start wait of local node l, for directed and undirected graphs alike.
//  1. threads 0..deg-1: every rank owning an in-neighbor of l in graph `gid` has published round k; with the sequence
//     check enabled, also verify that the row about to be read is tagged with round k.
//  2. threads 32.. (k > 0): every rank owning a round-(k-1) reader of l has published round k.  Node l overwrites
//     pub[(k+1)&1] at the end of round k, the buffer its round-(k-1) readers read during round k-1.  A rank publishes
//     round k only after its round-(k-1) reads, so this wait closes the write-after-read window without a separate
//     "consumed" counter (tests/test_protocol_model.py, tests/test_protocol_model_directed.py).
// The readers of l are its out-neighbors.  With a directed graph in the plan they are not the nodes l pulls from and
// come from the reader tables (rdr_deg, rdr_rank).  Without reader tables every graph is undirected, the readers are
// the neighbors of graph_id[k-1], and step 2 is skipped when that graph is `gid`: step 1 waited for the same ranks.
// (Step 2 picks the rank in two branches and waits once: with the table pointers selected first,
// dinno_update_kernel<double, 16> compiled to 246 registers instead of 168.)
template <typename T>
NNDT_DEVINL void wait_neighbors(const Common<T>& c, int gid, int l, int k) {
  const bool check = c.nbr_seq != nullptr;
  if (c.world > 1 || check) {
    const int d = c.deg[gid * c.L + l];
    if ((int)threadIdx.x < d) {
      const int r = c.world > 1 ? c.nbr_rank[(gid * c.L + l) * c.dmax + threadIdx.x] : -1;
      if (r >= 0) wait_rank(c, r, k);
      if (check) {
        const int* tag = reinterpret_cast<const int*>(c.nbr_seq[((size_t)(gid * c.L + l) * c.dmax + threadIdx.x) * 2 + (k & 1)]);
        if (ld_acquire_sys(tag) != k) *c.err = 2;
      }
    }
    if (c.world > 1 && k > 0) {
      const int gp = c.graph_id[k - 1], t = (int)threadIdx.x - 32;   // a different warp than the in-neighbor waiters
      int r = -1;
      if (c.rdr_deg != nullptr) {
        if (t >= 0 && t < c.rdr_deg[gp * c.L + l]) r = c.rdr_rank[(gp * c.L + l) * c.rmax + t];
      } else if (gp != gid) {
        if (t >= 0 && t < c.deg[gp * c.L + l]) r = c.nbr_rank[(gp * c.L + l) * c.dmax + t];
      }
      if (r >= 0) wait_rank(c, r, k);
    }
    __syncthreads();
  }
}

// tag the rows published for round k + 1 (one thread per node, before the launch's arrival counter)
template <typename T>
NNDT_DEVINL void tag_published(const Common<T>& c, int l, int k) {
  if (c.pub_seq != nullptr && blockIdx.x == 0 && threadIdx.x == 0) c.pub_seq[((k + 1) & 1) * c.pub_L + l] = k + 1;
}

// tell the peers that every round below `kn` is published (called by threads 0..world-1 of ONE block after the rows are
// ordered before this point at gpu scope): one remote store per rank that ever owns a neighbor
template <typename T>
NNDT_DEVINL void announce_round(const Common<T>& c, int kn) {
  __threadfence_system();
  if ((int)threadIdx.x < c.world && (int)threadIdx.x != c.rank && ((c.notify_mask >> threadIdx.x) & 1ull))
    st_release_sys(reinterpret_cast<int*>(c.peer_flag[threadIdx.x]), kn);
}

// First consensus kernel of round k (the one that reads neighbor rows).  Block (0, 0) announces "round k published"
// here rather than at the end of round k - 1's final kernel: that kernel wrote the rows, it is complete and flushed by
// the time any block of this one runs (every kernel passes griddepcontrol.wait before it lets its dependents launch),
// and the system fence + NVLink flag stores (3-4 us when they sit at the end of a kernel the next forward/backward
// waits for) overlap the forward/backward kernel this launch runs under.
template <typename T>
NNDT_DEVINL void begin_round(const Common<T>& c, int gid, int l, int k) {
  if (c.world > 1 && blockIdx.x == 0 && blockIdx.y == 0) announce_round(c, k);
  if (c.sum_mode) wait_all_sums(c, k); else wait_neighbors(c, gid, l, k);
}

// last block of the launch: advance the round counter (the next round's first kernel announces it to the peers)
template <typename T>
NNDT_DEVINL void finish_round(const Common<T>& c, int k) {
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned total = gridDim.x * gridDim.y;
    is_last = (atomicAdd(c.done_ctr, 1u) == total - 1);
  }
  __syncthreads();
  if (is_last) {
    if (threadIdx.x == 0) {
      *c.done_ctr = 0;
      *c.round_ctr = k + 1;
    }
  }
}

template <typename T>
NNDT_DEVINL const T* nbr_row(const Common<T>& c, int gid, int l, int e, int par, int chan) {
  return reinterpret_cast<const T*>(c.nbr_ptr[(((size_t)(gid * c.L + l) * c.dmax + e) * 2 + par) * c.C + chan]);
}

// Pull the neighbors' values at this thread's element: up to D neighbor rows in flight per thread, load(e) for each
// before acc(e, value) combines any, in neighbor order.  Over NVLink a load is ~2 us; issued one by one they add up.
template <int D, class FL, class FA>
NNDT_DEVINL void for_neighbors(int deg, FL load, FA acc) {
  for (int e0 = 0; e0 < deg; e0 += D) {
    decltype(load(0)) q[D];
#pragma unroll
    for (int j = 0; j < D; ++j)
      if (e0 + j < deg) q[j] = load(e0 + j);
#pragma unroll
    for (int j = 0; j < D; ++j)
      if (e0 + j < deg) acc(e0 + j, q[j]);
  }
}

template <typename T>
NNDT_DEVINL T* pub_row(const Common<T>& c, int par, int chan, int l) {
  return c.pub + ((size_t)(par * c.C + chan) * c.pub_L + l) * c.n_pad;
}

// ---- complete-graph mode -----------------------------------------------------------------------
// network-wide sum of channel `chan` at element i for parity `par`
template <int N> struct DPack { double v[N]; };
template <typename T>
NNDT_DEVINL DPack<Vec<T>::N> network_sum(const Common<T>& c, int par, int chan, int i) {
  constexpr int N = Vec<T>::N;
  const size_t off = (size_t)(par * c.C + chan) * c.n_pad + i;
  DPack<N> r;
  if (c.sum_mc != nullptr) {
#pragma unroll
    for (int u = 0; u < N; ++u)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f64 %0, [%1];" : "=d"(r.v[u]) : "l"(c.sum_mc + off + u) : "memory");
  } else {
#pragma unroll
    for (int u = 0; u < N; u += 2) {
      const double2 q = *reinterpret_cast<const double2*>(c.sum_local + off + u);
      r.v[u] = q.x; r.v[u + 1] = q.y;
    }
  }
  return r;
}
// every rank's partial sum of round k must be in place before the in-switch reduction reads it
template <typename T>
NNDT_DEVINL void wait_all_sums(const Common<T>& c, int k) {
  if (c.world > 1) {
    if ((int)threadIdx.x < c.world && (int)threadIdx.x != c.rank) {
      const long long t0 = clock64();
      while (ld_acquire_sys(c.sum_flags + threadIdx.x) < k + 1) {
        if (clock64() - t0 > kSpinLimit) { *c.err = 1; break; }
      }
    }
    __syncthreads();
  }
}

// ---- Gossip-PGA: round k is global when k mod period == period - 1 ----
// `sum_par` is the parity of the partial-sum buffer of global round k: the parity of the global round's count
// g = k / period, not of k.
// Round parity is unsafe once global rounds are `period` apart: with an even period every global round lands on the
// same parity, and a rank more than period - 1 gossip hops ahead could overwrite its partial of global round g + 1
// while a far rank still reduces g (tests/test_protocol_model_pga.py finds that interleaving at period 2 on a 3-rank
// path).  With the count's parity, a rank writes its partial of g + 2 into g's buffer only after its global round g + 1
// waited for every rank's partial of g + 1, and each rank posts that partial only in round k_{g+1}, after every launch
// of round k_g, which read g's buffer, has completed.  So no rank still reads g's buffer when it is overwritten: the
// argument that makes the every-round complete-graph mode safe, applied to the global rounds alone.  The sum flags
// carry k + 1 and only grow, so "flag >= k + 1" is the same test in both modes.
struct PgaPhase { bool global; int sum_par; };
NNDT_DEVINL PgaPhase pga_phase(int k, int period) {
  const int g = k / period;
  return {k - g * period == period - 1, g & 1};
}

template <int U, typename T>
NNDT_DEVINL Pack<T> sum_partials(const Common<T>& c, int l, int i) {
  // all (up to U) partial loads are issued before the first add: one L2 round trip instead of S dependent ones;
  // the summation order stays s = 0, 1, 2, ...  (U = 4 for the cluster kernels' <= 4 partial rows per node: the
  // 16-deep variant costs 48 more registers and halves the occupancy of the update kernels)
  constexpr int N = Vec<T>::N;
  const T* gp = c.grad_part + (size_t)l * c.S * c.n_pad + i;
  Pack<T> q[U];
#pragma unroll
  for (int s = 0; s < U; ++s)
    if (s < c.S) q[s] = ldv(gp + (size_t)s * c.n_pad);
  Pack<T> g = q[0];
#pragma unroll
  for (int s = 1; s < U; ++s)
    if (s < c.S) {
#pragma unroll
      for (int u = 0; u < N; ++u) g.v[u] += q[s].v[u];
    }
  for (int s = U; s < c.S; ++s) {
    const Pack<T> r = ldv(gp + (size_t)s * c.n_pad);
#pragma unroll
    for (int u = 0; u < N; ++u) g.v[u] += r.v[u];
  }
  return g;
}

// sum_partials over any partial set: `gp` is the node's first partial row at element i, S rows n_pad apart; the same
// issue order and summation order s = 0, 1, 2, ...
template <int U, typename T>
NNDT_DEVINL Pack<T> sum_partial_rows(const T* gp, int S, int n_pad) {
  constexpr int N = Vec<T>::N;
  Pack<T> q[U];
#pragma unroll
  for (int s = 0; s < U; ++s)
    if (s < S) q[s] = ldv(gp + (size_t)s * n_pad);
  Pack<T> g = q[0];
#pragma unroll
  for (int s = 1; s < U; ++s)
    if (s < S) {
#pragma unroll
      for (int u = 0; u < N; ++u) g.v[u] += q[s].v[u];
    }
  for (int s = U; s < S; ++s) {
    const Pack<T> r = ldv(gp + (size_t)s * n_pad);
#pragma unroll
    for (int u = 0; u < N; ++u) g.v[u] += r.v[u];
  }
  return g;
}

// step bookkeeping done by one thread per node in the kernel that consumes a gradient: advance the sampler's
// draw counter and fold the step's training loss into the moving average (problems/dist_online_dense_problem.py:129-137)
template <typename T>
NNDT_DEVINL void step_bookkeeping(const Common<T>& c, int l) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (c.calls != nullptr) c.calls[l] += 1;
    if (c.tloss != nullptr) {
      float loss = 0.f;
      for (int s = 0; s < c.loss_S; ++s) loss += c.loss_part[l * c.loss_S + s];
      const float t = c.tloss[l];
      c.tloss[l] = t != 0.f ? (1.f - c.tdecay) * t + c.tdecay * loss : loss;
    }
  }
}

// End of a launch that consumes a gradient.  On the round's last step (`last`) it also tags the rows it published and
// then advances the round.  The order is part of the publication protocol: each block tags before it arrives at the
// launch's counter, so when the last arrival advances the round every node's rows of round k + 1 carry their tag.
template <typename T>
NNDT_DEVINL void end_step(const Common<T>& c, int l, int k, bool last) {
  step_bookkeeping(c, l);
  if (last) { tag_published(c, l, k); finish_round(c, k); }
}

// ---- torch.optim step on one vector: SGD, Adam (betas 0.9 / 0.999, eps 1e-8), AdamW (+ weight decay 0.01) ----
template <typename T>
struct OptCoef {
  T lr, step_size, bc2s;
  int opt;
};
// coefficients of optimizer step t (1-based, the torch.optim `step` count)
template <typename T>
NNDT_DEVINL OptCoef<T> opt_coef(int opt, T lr, int t) {
  OptCoef<T> q;
  q.lr = lr;
  const T bc1 = (T)1 - pow((T)0.9, (T)t);
  q.bc2s = sqrt((T)1 - pow((T)0.999, (T)t));
  q.step_size = q.lr / bc1;
  q.opt = opt;
  return q;
}
template <typename T>
NNDT_DEVINL void opt_apply(const OptCoef<T>& q, Pack<T>& th, Pack<T>& m, Pack<T>& v, const Pack<T>& g) {
  constexpr int N = Vec<T>::N;
  const T b1 = (T)0.9, b2 = (T)0.999, eps = (T)1e-8, wd = (T)1e-2;
  if (q.opt == kSGD) {
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] -= q.lr * g.v[u];
  } else {
#pragma unroll
    for (int u = 0; u < N; ++u) {
      if (q.opt == kAdamW) th.v[u] *= ((T)1 - q.lr * wd);
      m.v[u] = b1 * m.v[u] + ((T)1 - b1) * g.v[u];
      v.v[u] = b2 * v.v[u] + ((T)1 - b2) * g.v[u] * g.v[u];
      th.v[u] -= q.step_size * m.v[u] / (sqrt(v.v[u]) / q.bc2s + eps);
    }
  }
}

// ---- DiNNO arithmetic on one vector (optimizers/dinno.py:74-91): augmented-Lagrangian gradient + optimizer step ----
template <typename T>
struct DinnoCoef {
  OptCoef<T> o;
  T rho;
  int deg;
};
template <typename T>
NNDT_DEVINL DinnoCoef<T> dinno_coef(const DinnoArgs<T>& a, int k, int step, int deg) {
  DinnoCoef<T> q;
  q.rho = a.c.rho[k];
  const int t = a.persistent ? k * a.pits + step + 1 : step + 1;
  q.o = opt_coef(a.opt, a.c.lr[k], t);
  q.deg = deg;
  return q;
}
template <typename T>
NNDT_DEVINL void dinno_apply(const DinnoCoef<T>& q, Pack<T>& th, const Pack<T>& thk, const Pack<T>& dl, const Pack<T>& du,
                             Pack<T>& m, Pack<T>& v, const Pack<T>& gl) {
  constexpr int N = Vec<T>::N;
  Pack<T> g;
#pragma unroll
  for (int u = 0; u < N; ++u)
    g.v[u] = gl.v[u] + du.v[u] + (T)2 * q.rho * (T)q.deg * (th.v[u] - thk.v[u]) - q.rho * dl.v[u];
  opt_apply(q.o, th, m, v, g);
}

// ---- CHOCO code rows (layout in consensus.h) ----
// the products and quotients that make or decode a code are rounded on their own (never contracted into an FMA, and
// IEEE division under --use_fast_math), so ops/consensus_ref.py produces the same bytes
NNDT_DEVINL float mul_rn(float x, float y) { return __fmul_rn(x, y); }
NNDT_DEVINL double mul_rn(double x, double y) { return __dmul_rn(x, y); }
NNDT_DEVINL float div_rn(float x, float y) { return __fdiv_rn(x, y); }
NNDT_DEVINL double div_rn(double x, double y) { return __ddiv_rn(x, y); }
// correctly rounded square root (a plain sqrtf is an approximation under --use_fast_math)
NNDT_DEVINL float sqrt_rn(float x) { return __fsqrt_rn(x); }
NNDT_DEVINL double sqrt_rn(double x) { return __dsqrt_rn(x); }

template <typename T>
NNDT_DEVINL char* code_row(const ChocoArgs<T>& a, int par, int l) {
  return reinterpret_cast<char*>(a.c.pub) + ((size_t)par * a.c.C * a.c.pub_L + l) * (size_t)a.code_stride;
}
template <typename T>
NNDT_DEVINL const char* nbr_code_row(const ChocoArgs<T>& a, int gid, int l, int e, int par) {
  return reinterpret_cast<const char*>(nbr_row(a.c, gid, l, e, par, 0));
}

// dec(q) of the Vec<T>::N elements at i (i a multiple of N) of a code row; `lw` = live word of the block (sign only)
template <typename T, int Q>
NNDT_DEVINL Pack<T> choco_decode(const char* row, int n_pad, int i, unsigned lw) {
  constexpr int N = Vec<T>::N;
  Pack<T> d;
  if (Q == kCodeNone) {
    d = ldv(reinterpret_cast<const T*>(row) + i);
  } else if (Q == kCodeInt8) {
    const T sc = reinterpret_cast<const T*>(row + n_pad)[i >> 5];
    signed char q[N];
    if (N == 4) *reinterpret_cast<int*>(q) = *reinterpret_cast<const int*>(row + i);
    else *reinterpret_cast<short*>(q) = *reinterpret_cast<const short*>(row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) d.v[u] = mul_rn((T)q[u], sc);
  } else {
    const unsigned w = reinterpret_cast<const unsigned*>(row)[i >> 5];
    const T sc = reinterpret_cast<const T*>(row + (n_pad >> 3))[i >> 5];
#pragma unroll
    for (int u = 0; u < N; ++u) {
      const int b = (i & 31) + u;
      d.v[u] = ((lw >> b) & 1u) ? (((w >> b) & 1u) ? sc : -sc) : (T)0;
    }
  }
  return d;
}

// Q(v) of the Vec<T>::N elements at i, stored into the code row `out`; returns dec(Q(v)).  Every lane of the warp calls
// it: the G = 32 / N lanes holding one 32-element block reduce its scale with xor shuffles, and a lane past the end of
// the row (`in` false, v = 0) takes part in them and stores nothing.  The same arithmetic as the encoder written out in
// choco_step_kernel, which keeps its own copy: called through this function, its int8 variants compiled to a different
// instruction schedule (same instruction count).
template <typename T, int Q>
NNDT_DEVINL Pack<T> choco_encode(const Pack<T>& v, char* out, int n_pad, int i, bool in, int lane, const unsigned* live) {
  constexpr int N = Vec<T>::N;
  constexpr int G = 32 / N;
  Pack<T> d;
  const bool head = (lane & (G - 1)) == 0;      // the lane that stores the block's scale / sign word
  if (Q == kCodeNone) {
    d = v;
    if (in) stv(reinterpret_cast<T*>(out) + i, v);
  } else if (Q == kCodeInt8) {
    T m = (T)0;
#pragma unroll
    for (int u = 0; u < N; ++u) m = fmax(m, fabs(v.v[u]));
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    const T sc = div_rn(m, (T)127);
    signed char q[N];
#pragma unroll
    for (int u = 0; u < N; ++u) {
      const T r = sc > (T)0 ? rint(div_rn(v.v[u], sc)) : (T)0;
      q[u] = (signed char)fmin(fmax(r, (T)-127), (T)127);
      d.v[u] = mul_rn((T)q[u], sc);
    }
    if (in) {
      if (N == 4) *reinterpret_cast<int*>(out + i) = *reinterpret_cast<const int*>(q);
      else *reinterpret_cast<short*>(out + i) = *reinterpret_cast<const short*>(q);
      if (head) reinterpret_cast<T*>(out + n_pad)[i >> 5] = sc;
    }
  } else {
    const unsigned lw = in ? live[i >> 5] : 0u;
    // sum |v| over the live elements: in element order within the lane, then halving across the block's lanes
    T p = (T)0;
    unsigned bits = 0u;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      const int b = (i & 31) + u;
      const T av = ((lw >> b) & 1u) ? fabs(v.v[u]) : (T)0;
      p = u == 0 ? av : p + av;
      if (v.v[u] >= (T)0) bits |= 1u << b;
    }
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) {
      p += __shfl_xor_sync(0xffffffffu, p, o);
      bits |= __shfl_xor_sync(0xffffffffu, bits, o);
    }
    const int nl = __popc(lw);
    const T sc = nl > 0 ? div_rn(p, (T)nl) : (T)0;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      const int b = (i & 31) + u;
      d.v[u] = ((lw >> b) & 1u) ? (((bits >> b) & 1u) ? sc : -sc) : (T)0;
    }
    if (in && head) {
      reinterpret_cast<unsigned*>(out)[i >> 5] = bits;
      reinterpret_cast<T*>(out + (n_pad >> 3))[i >> 5] = sc;
    }
  }
  return d;
}

// ---- BEER (layout in consensus.h): code row of channel `chan` (0: theta - h, 1: v - g) ----
template <typename T>
NNDT_DEVINL char* beer_code_row(const BeerArgs<T>& a, int par, int chan, int l) {
  const Common<T>& c = a.c;
  return reinterpret_cast<char*>(c.pub) + ((size_t)(par * c.C + chan) * c.pub_L + l) * (size_t)a.code_stride;
}

// ---- top-k code rows (layout in consensus.h) ----
// the slice of the row one CTA of the step's cluster owns: a multiple of 32 elements, so every slice starts 16-byte
// aligned and holds whole live words
__host__ __device__ __forceinline__ int topk_slice(int n_pad) {
  return ((n_pad + kTopkCluster - 1) / kTopkCluster + 31) / 32 * 32;
}

// selection keys: the IEEE bits with the sign bit cleared, as an unsigned integer ordered as |v|
template <typename T> struct TopkKey;
template <> struct TopkKey<float> {
  using K = unsigned;
  static constexpr int kPasses = 4;                 // 31 key bits, 8-bit digits from bit 24 down
  static NNDT_DEVINL K key(float v) { return __float_as_uint(v) & 0x7fffffffu; }
};
template <> struct TopkKey<double> {
  using K = unsigned long long;
  static constexpr int kPasses = 8;                 // 63 key bits, 8-bit digits from bit 56 down
  static NNDT_DEVINL K key(double v) { return (unsigned long long)__double_as_longlong(v) & 0x7fffffffffffffffull; }
};

constexpr int kTopkBins = 256;                      // one 8-bit digit; THREADS == kTopkBins: a thread per bin
struct TopkShared {
  unsigned hist[2][kTopkBins];                      // this CTA's digit histograms, double buffered (peers read them)
  unsigned tot[kTopkBins];                          // the cluster's sums of the current pass
  unsigned long long cta_cnt[2];                    // per channel: (above << 32) | equal keys of this CTA (peers read)
  unsigned long long warp_cnt[THREADS / 32];
  int bin, kr, cnt;                                 // the digit a pass picked, the entries still to take, its bin count
};

// the k-th largest key so far: keys k with (k & mask) > prefix are selected, and of those equal to prefix the first kr
template <typename T>
struct TopkThr {
  typename TopkKey<T>::K prefix, mask;
  int kr;
};

// live bit of slice element j: `live` is the slice's copy of the mask in shared memory (slices start on a word)
NNDT_DEVINL bool live_at(const unsigned* live, int j) { return (live[j >> 5] >> (j & 31)) & 1u; }

// copy the live words of the slice [base, base + len) into shared memory
NNDT_DEVINL void topk_live_words(unsigned* dst, const unsigned* live, int base, int len) {
  for (int w = threadIdx.x; w < (len >> 5); w += THREADS) dst[w] = live[(base >> 5) + w];
}

// MSD radix select over the cluster: sv [len] is this CTA's slice and `live` its live words in shared memory; every CTA
// of the cluster calls it and gets the same result.  Each pass counts this CTA's live keys that match the prefix so far per 8-bit digit (warp
// aggregated shared atomics), sums the cluster's histograms through DSMEM and picks the digit where the count from the
// top reaches kr.  It stops early when that digit's bin holds exactly kr keys: all of them are selected and no tie is
// left.  `pc` counts passes over the channels of a launch: the histograms are double buffered, so the one cluster
// barrier of a pass also guarantees that the peers have read the buffer it zeroes (they read it two passes back).
template <typename T>
NNDT_DEVINL TopkThr<T> topk_threshold(const T* sv, int len, const unsigned* live, int k, TopkShared& sh, int& pc) {
  using KT = TopkKey<T>;
  using K = typename KT::K;
  TopkThr<T> r;
  r.prefix = 0; r.mask = 0; r.kr = k;
  for (int p = 0; p < KT::kPasses; ++p) {
    const int shift = 8 * (KT::kPasses - 1 - p);
    unsigned* h = sh.hist[pc & 1];
    ++pc;
    h[threadIdx.x] = 0u;
    __syncthreads();
    for (int j = threadIdx.x; j < len; j += THREADS) {     // len is a multiple of 32: whole warps iterate
      int bin = -1;
      if (live_at(live, j)) {
        const K key = KT::key(sv[j]);
        if ((key & r.mask) == r.prefix) bin = (int)(key >> shift) & (kTopkBins - 1);
      }
      const unsigned same = __match_any_sync(0xffffffffu, bin);
      if (bin >= 0 && (int)(threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(&h[bin], (unsigned)__popc(same));
    }
    cluster_sync();
    unsigned part[kTopkCluster], t = 0u;          // all loads in flight before the first add
#pragma unroll
    for (int q = 0; q < kTopkCluster; ++q) part[q] = ld_dsmem_u32(map_to(h + threadIdx.x, q));
#pragma unroll
    for (int q = 0; q < kTopkCluster; ++q) t += part[q];
    sh.tot[threadIdx.x] = t;
    __syncthreads();
    if (threadIdx.x < 32) {
      // lane holds bins 8 lane .. 8 lane + 7; `above` counts the keys in the bins of the higher lanes
      const int lane = threadIdx.x;
      unsigned cnt[8], s = 0u;
#pragma unroll
      for (int u = 0; u < 8; ++u) { cnt[u] = sh.tot[8 * lane + u]; s += cnt[u]; }
      unsigned suf = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned x = __shfl_down_sync(0xffffffffu, suf, o);
        if (lane + o < 32) suf += x;
      }
      unsigned cum = suf - s;
      if (cum < (unsigned)r.kr && (unsigned)r.kr <= suf) {
        for (int u = 7; u >= 0; --u) {
          if (cum + cnt[u] >= (unsigned)r.kr) {
            sh.bin = 8 * lane + u; sh.kr = r.kr - (int)cum; sh.cnt = (int)cnt[u];
            break;
          }
          cum += cnt[u];
        }
      }
    }
    __syncthreads();
    r.prefix |= (K)sh.bin << shift;
    r.mask |= (K)(kTopkBins - 1) << shift;
    r.kr = sh.kr;
    if (sh.cnt == r.kr) break;
  }
  return r;
}

// Position of every selected entry of the slice in the code row, index order: thread t walks the contiguous segment
// t of the slice; a block scan and a cluster exclusive scan of the packed (above, equal) counts give the entries
// before it.  emit(j, pos) is called once per selected slice element j.
template <typename T, class F>
NNDT_DEVINL void topk_emit(const T* sv, int len, const unsigned* live, const TopkThr<T>& thr, TopkShared& sh, int ch,
                           F emit) {
  using KT = TopkKey<T>;
  using K = typename KT::K;
  const int seg = (len + THREADS - 1) / THREADS;
  const int j0 = min(len, (int)threadIdx.x * seg), j1 = min(len, j0 + seg);
  unsigned gt = 0u, eq = 0u;
  for (int j = j0; j < j1; ++j) {
    if (!live_at(live, j)) continue;
    const K mk = KT::key(sv[j]) & thr.mask;
    gt += mk > thr.prefix;
    eq += mk == thr.prefix;
  }
  const unsigned long long mine = ((unsigned long long)gt << 32) | eq;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long x = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += x;
  }
  if (lane == 31) sh.warp_cnt[wid] = incl;
  __syncthreads();
  unsigned long long before = incl - mine, cta = 0ull;
  for (int w = 0; w < THREADS / 32; ++w) {
    const unsigned long long x = sh.warp_cnt[w];
    if (w < wid) before += x;
    cta += x;
  }
  if (threadIdx.x == 0) sh.cta_cnt[ch] = cta;
  cluster_sync();
  const unsigned rank = cluster_rank();
  for (unsigned q = 0; q < rank; ++q) before += ld_dsmem_u64(map_to(&sh.cta_cnt[ch], q));
  unsigned gtb = (unsigned)(before >> 32), eqb = (unsigned)before;
  const unsigned kr = (unsigned)thr.kr;
  for (int j = j0; j < j1; ++j) {
    if (!live_at(live, j)) continue;
    const K mk = KT::key(sv[j]) & thr.mask;
    if (mk > thr.prefix) {
      emit(j, gtb + min(eqb, kr));
      ++gtb;
    } else if (mk == thr.prefix) {
      if (eqb < kr) emit(j, gtb + eqb);
      ++eqb;
    }
  }
}

// zero the bytes of a code row past its k entries (cluster rank 0 of the node)
NNDT_DEVINL void topk_pad(char* out, int k, int value_bytes, long long stride) {
  if (blockIdx.x != 0) return;
  for (long long b = (long long)k * (value_bytes + 4) + threadIdx.x; b < stride; b += THREADS) out[b] = 0;
}

// first j in [0, k) with idx[j] >= key (k when there is none), by the 32 lanes of a warp: each round probes 32 evenly
// spaced entries, so a row of k entries takes about log32(k) dependent loads
NNDT_DEVINL int warp_lower_bound(const unsigned* idx, int k, unsigned key, int lane) {
  int lo = 0, hi = k;                               // the answer lies in [lo, hi]
  while (lo < hi) {
    const int step = (hi - lo + 31) >> 5;
    const int p = lo + lane * step;
    const unsigned m = __ballot_sync(0xffffffffu, p >= hi || idx[p] >= key);
    if (m == 0u) { lo += 31 * step + 1; continue; }
    const int f = __ffs(m) - 1;
    if (f == 0) break;
    hi = min(hi, lo + f * step);
    lo += (f - 1) * step + 1;
  }
  return lo;
}

// scatter the entries of a top-k code row that fall in the elements [c0, c0 + len) into tile [len] (zeroed by the
// caller), by one warp
template <typename T>
NNDT_DEVINL void topk_gather(const char* code, int k, int c0, int len, T* tile, int lane) {
  const T* vals = reinterpret_cast<const T*>(code);
  const unsigned* idx = reinterpret_cast<const unsigned*>(code + (size_t)k * sizeof(T));
  const int lo = warp_lower_bound(idx, k, (unsigned)c0, lane);
  const int hi = lo + warp_lower_bound(idx + lo, min(k - lo, len), (unsigned)(c0 + len), lane);
  for (int j = lo + lane; j < hi; j += 32) tile[idx[j] - c0] = vals[j];
}

// ---- ClippedGossip: chunks of THREADS * N elements, one distance partial each ----
template <typename T>
__host__ __device__ __forceinline__ int cg_chunks(const Common<T>& c) {
  return (c.n_pad + THREADS * Vec<T>::N - 1) / (THREADS * Vec<T>::N);
}

// ---- DP-DSGD (stream in consensus.h: DpArgs) ----
// the standard normals of elements 2p and 2p + 1 of stream (a, b) in round k: u1 in (0, 1] and u2 in [0, 1) from 53
// bits each, Box-Muller in fp64 (ops/consensus_ref.py: dp_normals)
NNDT_DEVINL double2 dp_normal2(unsigned key0, unsigned key1, unsigned p, unsigned k, unsigned a, unsigned b) {
  const uint4 x = curand_Philox4x32_10(make_uint4(p, k, a, b), make_uint2(key0, key1));
  const double u1 = (double)(((unsigned long long)(x.x >> 5) << 26) + (x.y >> 6) + 1ull) * 0x1p-53;
  const double u2 = (double)(((unsigned long long)(x.z >> 5) << 26) + (x.w >> 6)) * 0x1p-53;
  const double r = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi(2.0 * u2, &s, &c);
  return make_double2(r * c, r * s);
}

// v of node `me` at the Vec<T>::N elements from i: cz_dp xi_me + cz_pair sum_e s_e xi_{me, ids[e]} in fp64, the
// products rounded on their own as the host twin rounds them (ops/consensus_ref.py: dp_noise), 0 off the live elements,
// rounded once to T
template <typename T>
NNDT_DEVINL Pack<T> dp_noise(const DpArgs<T>& a, int k, unsigned me, int deg, const int* ids, int i) {
  constexpr int N = Vec<T>::N;
  const unsigned lw = a.live[i >> 5];
  Pack<T> out;
#pragma unroll
  for (int q = 0; q < N; q += 2) {
    const unsigned p = (unsigned)(i >> 1) + (unsigned)(q >> 1);
    double v0 = 0.0, v1 = 0.0;
    if (a.cz_dp != 0.0) {
      const double2 x = dp_normal2(a.key0, a.key1, p, (unsigned)k, me, kDpLocal);
      v0 = __dmul_rn(a.cz_dp, x.x);
      v1 = __dmul_rn(a.cz_dp, x.y);
    }
    if (a.cz_pair != 0.0 && deg > 0) {
      double e0 = 0.0, e1 = 0.0;
      for (int e = 0; e < deg; ++e) {
        const unsigned j = (unsigned)ids[e];
        const double2 x = dp_normal2(a.key0, a.key1, p, (unsigned)k, min(me, j), max(me, j));
        if (me < j) { e0 += x.x; e1 += x.y; } else { e0 -= x.x; e1 -= x.y; }
      }
      v0 += __dmul_rn(a.cz_pair, e0);
      v1 += __dmul_rn(a.cz_pair, e1);
    }
    const int b = (i & 31) + q;
    out.v[q] = ((lw >> b) & 1u) ? (T)v0 : (T)0;
    out.v[q + 1] = ((lw >> (b + 1)) & 1u) ? (T)v1 : (T)0;
  }
  return out;
}

// ---- Moniqua (layout and stream in consensus.h: MoniquaArgs) ----
template <typename T>
NNDT_DEVINL unsigned* mq_code_row(const MoniquaArgs<T>& a, int par, int l) {
  return reinterpret_cast<unsigned*>(reinterpret_cast<char*>(a.c.pub) + ((size_t)par * a.c.pub_L + l) * (size_t)a.code_stride);
}

// the codes of the Vec<T>::N elements from i in the low bits of the result (element i + u at bits u * BITS)
template <typename T, int BITS>
NNDT_DEVINL unsigned mq_word(const unsigned* row, int i) {
  return row[(i * BITS) >> 5] >> ((i * BITS) & 31);
}

// the code of x (fp64) rounded with the 32 random bits r; every operation a single IEEE one, as mq_codes
template <int BITS>
NNDT_DEVINL unsigned mq_code(double x, double B, unsigned r) {
  const double z = __ddiv_rn(x, B);
  const double t = __dmul_rn(__dsub_rn(z, floor(z)), (double)(1 << BITS));
  const double fl = floor(t);
  const double u = __dmul_rn((double)r, 0x1p-32);
  return ((unsigned)fl + (u < __dsub_rn(t, fl) ? 1u : 0u)) & ((1u << BITS) - 1u);
}

// xhat of code c from yb = y / B, and the margin offset v - n
template <int BITS>
NNDT_DEVINL double mq_decode(unsigned c, double yb, double B, double& off) {
  const double cl = (double)c * (1.0 / (1 << BITS));       // exact
  const double v = __dsub_rn(yb, cl);
  const double n = rint(v);
  off = __dsub_rn(v, n);
  return __dmul_rn(B, __dadd_rn(cl, n));
}

// ---- SPARQ-SGD (layout in consensus.h: SparqArgs) ----
template <typename T>
NNDT_DEVINL char* sparq_row(const SparqArgs<T>& a, int par, int l) {
  return reinterpret_cast<char*>(a.c.pub) + ((size_t)par * a.c.pub_L + l) * (size_t)a.row_stride;
}
// the trigger bit in the tail of a published row
NNDT_DEVINL bool sparq_trig(const char* row, long long code_bytes) {
  return *reinterpret_cast<const unsigned*>(row + code_bytes) != 0u;
}

// ---- SGP (layout in consensus.h) ----
template <typename T>
NNDT_DEVINL T* sgp_row(const SgpArgs<T>& a, int par, int l) {
  return reinterpret_cast<T*>(reinterpret_cast<char*>(a.c.pub) + ((size_t)par * a.c.pub_L + l) * (size_t)a.row_stride);
}
// the float64 push-sum weight in the tail of a published row
template <typename T>
NNDT_DEVINL double row_weight(const T* row, int n_pad) {
  return *reinterpret_cast<const double*>(row + n_pad);
}
// theta = x / w: w rounded to T, then one IEEE division (ops/consensus_ref.py: sgp_debias)
template <typename T>
NNDT_DEVINL T sgp_debias(T x, double w) {
  return div_rn(x, (T)w);
}

// ---- Push-DIGing (layout in consensus.h): row of channel `chan` (0: u with the w tail, 1: y) ----
template <typename T>
NNDT_DEVINL T* pdg_row(const PushDigArgs<T>& a, int par, int chan, int l) {
  const Common<T>& c = a.c;
  return reinterpret_cast<T*>(reinterpret_cast<char*>(c.pub) + ((size_t)(par * c.C + chan) * c.pub_L + l) * (size_t)a.row_stride);
}

}  // namespace consensus
}  // namespace nndt
