// Fused neighbor-exchange + mixing + optimizer-update kernels for DiNNO / DSGD / DSGD with momentum / DSGT /
// Exact Diffusion / CHOCO-SGD / BEER / SGP / Push-DIGing.
//
// Reference call sites replaced (all Python loops over nodes x parameter tensors):
//   optimizers/dinno.py:103-125 + :74-91  -> dinno_update   (exchange, dual ascent, prox-grad, Adam/SGD/AdamW)
//   optimizers/dsgd.py:37-46 / :55-58      -> dsgd_mix / dsgd_step
//   optimizers/dsgt.py:58-75 / :87-103     -> dsgt_mix / dsgt_track
// Exact Diffusion (no reference counterpart, optimizers/exact_diffusion.py) -> dsgd_mix or ed_sum_mix / ed_step
// DSGD with momentum (no reference counterpart, optimizers/dsgdm.py)       -> dsgd_mix / dsgdm_step
// CHOCO-SGD (no reference counterpart, optimizers/choco.py)                -> choco_mix / choco_step
//                                                          (top-k codes)   -> choco_topk_mix / choco_topk_step
// BEER (no reference counterpart, optimizers/beer.py)                      -> beer_mix / beer_step
//                                                          (top-k codes)   -> beer_topk_mix / beer_topk_step
// K-GT / local DSGD (no reference counterpart, optimizers/kgt.py)          -> kgt_mix or dsgd_mix / K x kgt_step
// DeTAG (no reference counterpart, optimizers/detag.py)                    -> K x ag_gossip / detag_track
// GT-HSGD (no reference counterpart, optimizers/gt_hsgd.py)                -> dsgt_mix / hsgd_track
// cross-gradient (no reference counterpart, optimizers/cross_gradient.py)  -> xg_pull / xg_publish, xg_step
// Gossip-PGA / local SGD (no reference counterpart, optimizers/gossip_pga.py) -> pga_sum + pga_mix / dsgd_step
// SlowMo (no reference counterpart, optimizers/slowmo.py)  -> pga_sum + pga_mix + slowmo_outer / dsgd_step or dsgdm_step
// DP-DSGD / DECOR (no reference counterpart, optimizers/dp_dsgd.py)        -> dsgd_mix / dp_norm + dp_step
// Moniqua (no reference counterpart, optimizers/moniqua.py)                -> mq_mix / mq_step
// decentralized AMSGrad / AdaGrad (no reference counterpart,
//                                  optimizers/dadaptive.py)                -> dadaptive_mix or dsgd_mix / dadaptive_step
// RelaySum (no reference counterpart, optimizers/relaysum.py)             -> relay_mix / relay_step
// ClippedGossip (no reference counterpart, optimizers/clipped_gossip.py)   -> cg_dist + cg_mix or dsgd_mix / cg_step
// BRIDGE (no reference counterpart, optimizers/bridge.py)                  -> bridge_mix / cg_step
// PowerGossip (no reference counterpart, optimizers/powergossip.py)        -> pg_mix / pg_step
// SGP (no reference counterpart, optimizers/sgp.py)                        -> sgp_mix / sgp_step
// Push-DIGing (no reference counterpart, optimizers/push_diging.py)        -> pdg_mix / pdg_track
//
// Every kernel is a single pass over the node's 16-byte vectorised parameter row: neighbor
// rows are pulled straight from the (local or NVLink-peer) published buffers named by the
// pointer table, combined with the Metropolis row in registers, the gradient partials of the
// forward/backward kernel are summed on the fly, the optimizer update is applied and the new
// row is published — no [d_i, n] stack, no cdist, no separate reduce or elementwise launch.
//
// Cross-GPU protocol (pull model): published rows are double buffered by round parity.  A
// rank announces "round k published" by writing k into its slot of every peer's flag array
// (st.release.sys over NVLink after __threadfence_system()); consumers spin with
// ld.acquire.sys on their *local* flag array only for the ranks that own a neighbor.  Since a
// node publishes k+1 only after finishing its round-k reads, two buffers suffice.
#include <mutex>
#include <unordered_map>

#include "consensus_device.cuh"

namespace nndt {
namespace consensus {

// S_local[par][chan] = sum over this rank's nodes of the published rows of round k
template <typename T>
__global__ void __launch_bounds__(THREADS) local_sum_kernel(const Common<T> c) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int N = Vec<T>::N;
  const RoundInfo<T> ri = round_info(c);
  for (int ch = 0; ch < c.C; ++ch) {
    for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
      double s[N];
#pragma unroll
      for (int u = 0; u < N; ++u) s[u] = 0.0;
      for (int l = 0; l < c.L; ++l) {
        const Pack<T> q = ldv(pub_row(c, ri.par, ch, l) + i);
#pragma unroll
        for (int u = 0; u < N; ++u) s[u] += (double)q.v[u];
      }
      double* dst = c.sum_local + (size_t)(ri.par * c.C + ch) * c.n_pad + i;
#pragma unroll
      for (int u = 0; u < N; u += 2) *reinterpret_cast<double2*>(dst + u) = make_double2(s[u], s[u + 1]);
    }
  }
  // last block: tell every peer that this rank's partial sum of round k is ready
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(c.done_ctr, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last) {
    if (threadIdx.x == 0) *c.done_ctr = 0;
    if (c.world > 1) {
      __threadfence_system();
      if ((int)threadIdx.x < c.world && (int)threadIdx.x != c.rank)
        st_release_sys(reinterpret_cast<int*>(c.peer_sum_flag[threadIdx.x]), ri.k + 1);
    }
  }
}


// ------------------------------------------------------------------ DiNNO ----
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) dinno_update_kernel(const DinnoArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  const DinnoCoef<T> cf = dinno_coef(a, ri.k, a.step, deg);
  const T rho = cf.rho;
  const bool first = a.step == 0, last = a.step == a.pits - 1;
  tl_stamp(c, ri.k, a.step, 0);
  if (first) begin_round(c, ri.gid, l, ri.k);
  tl_stamp(c, ri.k, a.step, 1);

  const bool fresh = first && !a.persistent;  // Adam moments restart every round (reference Q3)

  const size_t row = (size_t)l * c.n_pad;
  const T* thk_row = pub_row(c, ri.par, 0, l);
  // The grid covers the row exactly once (one vector per thread), so all state that the preceding
  // forward/backward kernel does not write is fetched BEFORE the programmatic-dependency wait and
  // overlaps that kernel's tail; only the gradient partials are read after it.
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    Pack<T> thk, dl, du;
    if (first) {
      thk = th;  // live row == theta^k at round start
#pragma unroll
      for (int u = 0; u < N; ++u) dl.v[u] = (T)0;
      if (c.sum_mode) {   // delta = S_all - N theta_i   (every other node is a neighbor)
        const DPack<N> sall = network_sum(c, ri.par, 0, i);
#pragma unroll
        for (int u = 0; u < N; ++u) dl.v[u] = (T)(sall.v[u] - (double)c.n_total * (double)thk.v[u]);
      } else {
        // for_neighbors<4> written out: through the helper's lambdas this kernel compiles to a different stream
        for (int e0 = 0; e0 < deg; e0 += 4) {
          Pack<T> q[4];
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (e0 + j < deg) q[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (e0 + j < deg) {
#pragma unroll
              for (int u = 0; u < N; ++u) dl.v[u] += q[j].v[u] - thk.v[u];
            }
        }
      }
      du = ldv(a.dual + row + i);
#pragma unroll
      for (int u = 0; u < N; ++u) du.v[u] -= rho * dl.v[u];
      stv(a.delta + row + i, dl);
      stv(a.dual + row + i, du);
    } else {
      thk = ldv(thk_row + i);
      dl = ldv(a.delta + row + i);
      du = ldv(a.dual + row + i);
    }
    Pack<T> m, v;
    if (a.opt != kSGD) {
      if (fresh) {
#pragma unroll
        for (int u = 0; u < N; ++u) { m.v[u] = (T)0; v.v[u] = (T)0; }
      } else {
        m = ldv(a.m + row + i);
        v = ldv(a.v + row + i);
      }
    }
    if (!waited) { tl_stamp(c, ri.k, a.step, 2); release_dependents_once(waited); tl_stamp(c, ri.k, a.step, 3); }
    const Pack<T> gl = sum_partials<U>(c, l, i);
    dinno_apply(cf, th, thk, dl, du, m, v, gl);
    if (a.opt != kSGD) {
      stv(a.m + row + i, m);
      stv(a.v + row + i, v);
    }
    stv(c.theta + row + i, th);
    if (last) stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
  }
  release_dependents_once(waited);
  tl_stamp(c, ri.k, a.step, 4);
  end_step(c, l, ri.k, last);
}

// ------------------------------------------------------------- local step ----
// One optimizer step per node that has not used up its budget; a node at its budget is left bitwise untouched (theta,
// moments, calls).  The forward/backward kernel before it has already run for every node, so a finished node's
// gradient is computed and dropped here.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) local_step_kernel(const LocalArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = blockIdx.y;
  // calls / budget / theta / moments were last written two launches back: readable before the dependency wait
  const int call = c.calls[l];
  if (call >= a.budget[l]) {
    pdl_wait();
    pdl_launch_dependents();
    return;
  }
  const OptCoef<T> q = opt_coef(a.opt, a.lr, call + 1);
  const size_t row = (size_t)l * c.n_pad;
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    Pack<T> m, v;
    if (a.opt != kSGD) {
      m = ldv(a.m + row + i);
      v = ldv(a.v + row + i);
    }
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    opt_apply(q, th, m, v, g);
    if (a.opt != kSGD) {
      stv(a.m + row + i, m);
      stv(a.v + row + i, v);
    }
    stv(c.theta + row + i, th);
  }
  release_dependents_once(waited);
  // the last CTA of node l to arrive advances its counter: every CTA has read `call` by then
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(a.arrive + l, 1u) == gridDim.x - 1) {
    a.arrive[l] = 0;
    c.calls[l] = call + 1;
  }
}

// ------------------------------------------------------------------- DSGD ----
template <typename T>
__global__ void __launch_bounds__(THREADS) dsgd_mix_kernel(const Common<T> c) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    if (c.sum_mode) {     // W = 11^T / N: the mixed row is the network mean
      const DPack<N> sall = network_sum(c, ri.par, 0, i);
      Pack<T> th;
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] = (T)(sall.v[u] / (double)c.n_total);
      stv(c.theta + row + i, th);
      continue;
    }
    Pack<T> th = ldv(c.theta + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] *= ws;
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i); },
                     [&](int e, const Pack<T>& q) {
#pragma unroll
                       for (int u = 0; u < N; ++u) th.v[u] += w[e] * q.v[u];
                     });
    stv(c.theta + row + i, th);
  }
}

template <typename T, int U>
__global__ void __launch_bounds__(THREADS) dsgd_step_kernel(const Common<T> c) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] -= alpha * g.v[u];
    stv(c.theta + row + i, th);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
  }
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------------- DSGT ----
// channel 0 of the published buffer is theta, channel 1 the gradient tracker y.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) dsgt_init_kernel(const DsgtArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> g = sum_partials<U>(c, l, i);
    stv(a.g_old + row + i, g);
    stv(pub_row(c, 0, 1, l) + i, g);
  }
  step_bookkeeping(c, l);
}

template <typename T, bool OWN>
__global__ void __launch_bounds__(THREADS) dsgt_mix_kernel(const DsgtArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T alpha = c.alpha[ri.k];
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const T* ys = pub_row(c, ri.par, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> al;                         // the step of each coordinate: the row, or alpha_k everywhere
    if (a.alpha_row != nullptr) {
      al = ldv(a.alpha_row + i);
    } else {
#pragma unroll
      for (int u = 0; u < N; ++u) al.v[u] = alpha;
    }
    if (c.sum_mode) {
      const DPack<N> st = network_sum(c, ri.par, 0, i);
      Pack<T> th;
      if (OWN) {                        // theta_i = S_theta / N - alpha (.) y_i
        const Pack<T> y = ldv(ys + i);
#pragma unroll
        for (int u = 0; u < N; ++u) th.v[u] = (T)(st.v[u] / (double)c.n_total) - al.v[u] * y.v[u];
      } else {                          // theta_i = (S_theta - alpha (.) S_y) / N
        const DPack<N> sy = network_sum(c, ri.par, 1, i);
#pragma unroll
        for (int u = 0; u < N; ++u) th.v[u] = (T)((st.v[u] - (double)al.v[u] * sy.v[u]) / (double)c.n_total);
      }
      stv(c.theta + row + i, th);
      continue;
    }
    Pack<T> th = ldv(c.theta + row + i);
    const Pack<T> y = ldv(ys + i);
    if (OWN) {
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] *= ws;
      // for_neighbors<2> written out, as below
      for (int e0 = 0; e0 < deg; e0 += 2) {
        Pack<T> q[2];
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if (e0 + j < deg) q[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if (e0 + j < deg) {
            const T we = w[e0 + j];
#pragma unroll
            for (int u = 0; u < N; ++u) th.v[u] += we * q[j].v[u];
          }
      }
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] -= al.v[u] * y.v[u];
      stv(c.theta + row + i, th);
      continue;
    }
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] = ws * (th.v[u] - al.v[u] * y.v[u]);
    // for_neighbors<2> written out: through the helper's lambdas this loop compiles to a different stream
    for (int e0 = 0; e0 < deg; e0 += 2) {
      Pack<T> qt[2], qy[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          qt[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
          qy[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 1) + i);
        }
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          const T we = w[e0 + j];
#pragma unroll
          for (int u = 0; u < N; ++u) th.v[u] += we * (qt[j].v[u] - al.v[u] * qy[j].v[u]);
        }
    }
    stv(c.theta + row + i, th);
  }
}

template <typename T, int U>
__global__ void __launch_bounds__(THREADS) dsgt_track_kernel(const DsgtArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const T* ys = pub_row(c, ri.par, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> y;
    if (c.sum_mode) {
      const DPack<N> sy = network_sum(c, ri.par, 1, i);
#pragma unroll
      for (int u = 0; u < N; ++u) y.v[u] = (T)(sy.v[u] / (double)c.n_total);
    } else {
      y = ldv(ys + i);
#pragma unroll
      for (int u = 0; u < N; ++u) y.v[u] *= ws;
      // for_neighbors<4> written out: through the helper's lambdas this kernel compiles to a different stream
      for (int e0 = 0; e0 < deg; e0 += 4) {
        Pack<T> q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < deg) q[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 1) + i);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < deg) {
            const T we = w[e0 + j];
#pragma unroll
            for (int u = 0; u < N; ++u) y.v[u] += we * q[j].v[u];
          }
      }
    }
    const Pack<T> gn = sum_partials<U>(c, l, i);
    const Pack<T> go = ldv(a.g_old + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) y.v[u] += gn.v[u] - go.v[u];
    stv(a.g_old + row + i, gn);
    stv(pub_row(c, ri.par ^ 1, 1, l) + i, y);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, ldv(c.theta + row + i));
  }
  end_step(c, l, ri.k, true);
}

// -------------------------------------------------------- Exact Diffusion ----
// The pointer-table mix is dsgd_mix_kernel fed with the weights of A = (I + W) / 2.  On the complete graph A's rows
// are (1/2) e_i + 1 / (2N), so the combine is (theta_i + S / N) / 2 with S the fp64 network sum.
template <typename T>
__global__ void __launch_bounds__(THREADS) ed_sum_mix_kernel(const Common<T> c) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  begin_round(c, ri.gid, l, ri.k);
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    const DPack<N> sall = network_sum(c, ri.par, 0, i);
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] = (T)(0.5 * ((double)th.v[u] + sall.v[u] / (double)c.n_total));
    stv(c.theta + row + i, th);
  }
}

// adapt psi' = theta - alpha_k g, correct theta <- psi' + (theta - psi), psi <- psi'; theta is published.  Round 0
// starts from psi = theta (the mixed row), so its step is plain DSGD.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) ed_step_kernel(const EdArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const bool init = ri.k == 0;
  const size_t row = (size_t)l * c.n_pad;
  // theta (written by the mix two launches back) and psi (the previous round's step) are read before the
  // programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> th = ldv(c.theta + row + i);
    Pack<T> dc;
    if (init) {
#pragma unroll
      for (int u = 0; u < N; ++u) dc.v[u] = (T)0;
    } else {
      const Pack<T> ps = ldv(a.psi + row + i);
#pragma unroll
      for (int u = 0; u < N; ++u) dc.v[u] = th.v[u] - ps.v[u];
    }
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    Pack<T> pn, tn;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      pn.v[u] = th.v[u] - alpha * g.v[u];
      tn.v[u] = pn.v[u] + dc.v[u];
    }
    stv(a.psi + row + i, pn);
    stv(c.theta + row + i, tn);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, tn);
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ---------------------------------------------------------- DSGD with momentum ----
// The mix is dsgd_mix_kernel.  The step, on the mixed row x (theta after the mix) with alpha_k from the schedule:
//   local (QG = false):   m <- beta m + g
//   quasi-global (QG):    mhat <- beta mhat + (1 - beta) (x_prev - x) / alpha_{k-1};  m = beta mhat + g;  x_prev <- x
//   theta <- x - alpha_k (NEST ? g + beta m : m);  theta is published.
// Round 0 reads neither the momentum row nor x_prev and takes them as zero (m = g, mhat = 0): its step is DSGD's.
// The 4-deep variant is held to 64 registers (4 CTAs per SM) without spilling; the quasi-global step's IEEE division
// otherwise takes it to 76 in fp64.  The deep variant keeps the compiler's choice (a minimum of 0 CTAs sets no limit).
template <typename T, int U, bool QG, bool NEST>
__global__ void __launch_bounds__(THREADS, U <= 4 ? 4 : 0) dsgdm_step_kernel(const MomentumArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const bool init = ri.k == 0;
  const T alpha_prev = QG && !init ? c.alpha[ri.k - 1] : (T)1;
  const T beta = a.beta, beta_c = (T)1 - a.beta;
  const size_t row = (size_t)l * c.n_pad;
  // theta (written by the mix two launches back), the momentum row and x_prev (the previous round's step) are read,
  // and mhat is advanced, before the programmatic-dependency wait; only the gradient partials of the forward/backward
  // kernel after it
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> x = ldv(c.theta + row + i);
    Pack<T> mb;                         // local: m of the previous round; quasi-global: mhat of this round
    if (init) {
#pragma unroll
      for (int u = 0; u < N; ++u) mb.v[u] = (T)0;
    } else {
      mb = ldv(a.m + row + i);
      if (QG) {
        const Pack<T> xp = ldv(a.x_prev + row + i);
#pragma unroll
        for (int u = 0; u < N; ++u) mb.v[u] = beta * mb.v[u] + beta_c * div_rn(xp.v[u] - x.v[u], alpha_prev);
      }
    }
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    Pack<T> m, th;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      m.v[u] = beta * mb.v[u] + g.v[u];
      th.v[u] = x.v[u] - alpha * (NEST ? g.v[u] + beta * m.v[u] : m.v[u]);
    }
    if (QG) {
      stv(a.m + row + i, mb);
      stv(a.x_prev + row + i, x);
    } else {
      stv(a.m + row + i, m);
    }
    stv(c.theta + row + i, th);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ---------------------------------------------------------------- CHOCO-SGD ----
// The published rows are code rows (consensus.h).  Round k: choco_mix reads the codes q^{k-1} of the node and its
// neighbors (all zero in round 0), s_i += W_ii dec(q_i) + sum_j W_ij dec(q_j), theta_i += gamma (s_i - x_hat_i);
// choco_step takes theta_i -= alpha_k g_i, q_i = Q(theta_i - x_hat_i), x_hat_i += dec(q_i) and publishes q_i.
template <typename T, int Q>
__global__ void __launch_bounds__(THREADS) choco_mix_kernel(const ChocoArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const char* own = code_row(a, ri.par, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const unsigned lw = Q == kCodeSign ? a.live[i >> 5] : 0u;
    Pack<T> t = choco_decode<T, Q>(own, c.n_pad, i, lw);
#pragma unroll
    for (int u = 0; u < N; ++u) t.v[u] *= ws;
    // the neighbor code rows are decoded in registers
    for_neighbors<4>(deg, [&](int e) { return choco_decode<T, Q>(nbr_code_row(a, ri.gid, l, e, ri.par), c.n_pad, i, lw); },
                     [&](int e, const Pack<T>& q) {
#pragma unroll
                       for (int u = 0; u < N; ++u) t.v[u] += w[e] * q.v[u];
                     });
    Pack<T> s = ldv(a.s + row + i);
    const Pack<T> xh = ldv(a.x_hat + row + i);
    Pack<T> th = ldv(c.theta + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) {
      s.v[u] += t.v[u];
      th.v[u] += a.gamma * (s.v[u] - xh.v[u]);
    }
    stv(a.s + row + i, s);
    stv(c.theta + row + i, th);
  }
}

// The G = 32 / N lanes holding one 32-element block reduce its scale with xor shuffles; the loop runs per warp, so
// every lane takes part, also the lanes past the end of a row shorter than a warp's span.
template <typename T, int U, int Q>
__global__ void __launch_bounds__(THREADS) choco_step_kernel(const ChocoArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  constexpr int G = 32 / N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  char* out = code_row(a, ri.par ^ 1, l);
  const int lane = threadIdx.x & 31;
  // theta (written by the mix two launches back) and x_hat (the previous round's step) are read before the
  // programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int w0 = (blockIdx.x * THREADS + (threadIdx.x & ~31)) * N; w0 < c.n_pad; w0 += gridDim.x * THREADS * N) {
    const int i = w0 + lane * N;
    const bool in = i < c.n_pad;
    Pack<T> th, xh;
#pragma unroll
    for (int u = 0; u < N; ++u) { th.v[u] = (T)0; xh.v[u] = (T)0; }
    if (in) {
      th = ldv(c.theta + row + i);
      xh = ldv(a.x_hat + row + i);
    }
    release_dependents_once(waited);
    Pack<T> v;
    if (in) {
      const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] -= alpha * g.v[u];
    }
#pragma unroll
    for (int u = 0; u < N; ++u) v.v[u] = th.v[u] - xh.v[u];
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
        if (head) reinterpret_cast<T*>(out + c.n_pad)[i >> 5] = sc;
      }
    } else {
      const unsigned lw = in ? a.live[i >> 5] : 0u;
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
        reinterpret_cast<T*>(out + (c.n_pad >> 3))[i >> 5] = sc;
      }
    }
    if (in) {
#pragma unroll
      for (int u = 0; u < N; ++u) xh.v[u] += d.v[u];
      stv(c.theta + row + i, th);
      stv(a.x_hat + row + i, xh);
    }
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------------- BEER ----
// Two channels of CHOCO code rows (consensus.h): channel 0 codes theta - h, channel 1 codes v - g.  Round k: beer_mix
// reads both codes of round k-1 of the node and its neighbors (all zero in round 0),
//   s_h_i += W_ii dec(qh_i) + sum_j W_ij dec(qh_j),  s_g_i += W_ii dec(qg_i) + sum_j W_ij dec(qg_j),
//   theta_i += gamma (s_h_i - h_i) - alpha v_i;
// beer_step takes v_i += gamma (s_g_i - g_i) + grad_i - m_old_i, m_old_i <- grad_i, qh_i = Q(theta_i - h_i),
// h_i += dec(qh_i), qg_i = Q(v_i - g_i), g_i += dec(qg_i) and publishes (qh_i, qg_i).  The tracker update sits in the
// step, beside the gradient it needs: folded into the mix it would move as many row loads as it saves and add a store.
template <typename T>
struct HGPack { Pack<T> h, g; };

template <typename T, int Q>
__global__ void __launch_bounds__(THREADS) beer_mix_kernel(const BeerArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T alpha = c.alpha[ri.k];
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const char* own_h = beer_code_row(a, ri.par, 0, l);
  const char* own_g = beer_code_row(a, ri.par, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const unsigned lw = Q == kCodeSign ? a.live[i >> 5] : 0u;
    Pack<T> th = choco_decode<T, Q>(own_h, c.n_pad, i, lw), tg = choco_decode<T, Q>(own_g, c.n_pad, i, lw);
#pragma unroll
    for (int u = 0; u < N; ++u) {
      th.v[u] *= ws;
      tg.v[u] *= ws;
    }
    // two neighbors' two code rows in flight, decoded in registers
    for_neighbors<2>(deg,
                     [&](int e) {
                       return HGPack<T>{
                           choco_decode<T, Q>(reinterpret_cast<const char*>(nbr_row(c, ri.gid, l, e, ri.par, 0)), c.n_pad, i, lw),
                           choco_decode<T, Q>(reinterpret_cast<const char*>(nbr_row(c, ri.gid, l, e, ri.par, 1)), c.n_pad, i, lw)};
                     },
                     [&](int e, const HGPack<T>& q) {
                       const T we = w[e];
#pragma unroll
                       for (int u = 0; u < N; ++u) {
                         th.v[u] += we * q.h.v[u];
                         tg.v[u] += we * q.g.v[u];
                       }
                     });
    Pack<T> sh = ldv(a.s_h + row + i), sg = ldv(a.s_g + row + i);
    const Pack<T> h = ldv(a.h + row + i), v = ldv(a.v + row + i);
    Pack<T> x = ldv(c.theta + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) {
      sh.v[u] += th.v[u];
      sg.v[u] += tg.v[u];
      x.v[u] += a.gamma * (sh.v[u] - h.v[u]) - alpha * v.v[u];
    }
    stv(a.s_h + row + i, sh);
    stv(a.s_g + row + i, sg);
    stv(c.theta + row + i, x);
  }
}

// Per-warp loop as in choco_step: both encoders reduce their blocks' scales with warp shuffles.
template <typename T, int U, int Q>
__global__ void __launch_bounds__(THREADS) beer_step_kernel(const BeerArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const size_t row = (size_t)l * c.n_pad;
  char* out_h = beer_code_row(a, ri.par ^ 1, 0, l);
  char* out_g = beer_code_row(a, ri.par ^ 1, 1, l);
  const int lane = threadIdx.x & 31;
  // theta and s_g (written by the mix two launches back), h, v, g and m_old (the previous round's step) are read
  // before the programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int w0 = (blockIdx.x * THREADS + (threadIdx.x & ~31)) * N; w0 < c.n_pad; w0 += gridDim.x * THREADS * N) {
    const int i = w0 + lane * N;
    const bool in = i < c.n_pad;
    Pack<T> x, h, v, g, sg, mo, gr;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      x.v[u] = (T)0; h.v[u] = (T)0; v.v[u] = (T)0; g.v[u] = (T)0; sg.v[u] = (T)0; mo.v[u] = (T)0; gr.v[u] = (T)0;
    }
    if (in) {
      x = ldv(c.theta + row + i);
      h = ldv(a.h + row + i);
      v = ldv(a.v + row + i);
      g = ldv(a.g + row + i);
      sg = ldv(a.s_g + row + i);
      mo = ldv(a.m_old + row + i);
    }
    release_dependents_once(waited);
    if (in) gr = sum_partials<U>(c, l, i);
    Pack<T> dx, dv;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      v.v[u] += a.gamma * (sg.v[u] - g.v[u]) + gr.v[u] - mo.v[u];
      dx.v[u] = x.v[u] - h.v[u];
      dv.v[u] = v.v[u] - g.v[u];
    }
    const Pack<T> qh = choco_encode<T, Q>(dx, out_h, c.n_pad, i, in, lane, a.live);
    const Pack<T> qg = choco_encode<T, Q>(dv, out_g, c.n_pad, i, in, lane, a.live);
    if (in) {
#pragma unroll
      for (int u = 0; u < N; ++u) {
        h.v[u] += qh.v[u];
        g.v[u] += qg.v[u];
      }
      stv(a.h + row + i, h);
      stv(a.v + row + i, v);
      stv(a.g + row + i, g);
      stv(a.m_old + row + i, gr);
    }
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------ top-k (CHOCO-SGD, BEER) ----
// kCodeTopk rows (consensus.h).  A code row holds only k entries, so neither kernel can work by position.
//
// The step runs one thread-block cluster of kTopkCluster CTAs per node, grid (CS, L): CTA r owns the contiguous slice
// [r sl, (r + 1) sl) of the row (topk_slice), so index order is (cluster rank, position in the slice).  It computes
// the dense step's arithmetic, keeps v in shared memory, selects with topk_threshold and writes the entries with
// topk_emit, and adds dec(q) = v to x_hat (BEER: h, g) at the selected indices only (x_hat is never -0, so x_hat + 0
// at the others would not change a bit).  A final cluster barrier keeps every CTA resident until its peers have read
// its shared memory.  The cluster has 8 CTAs, the portable size, which holds the PAPER MNIST row (n_pad 28 544) at
// 3 584 elements per CTA; 16 CTAs would need the non-portable attribute and double the DSMEM loads of every histogram
// reduction, and were not measured.  The digit is 8 bits: one bin per thread of the 256-thread CTA, so a histogram
// reduction is one DSMEM load per thread and peer, and a pass is one warp's scan of 256 bins.  On an H100 80GB HBM3
// (700 W) the step takes 25 us in fp64 against int8's 4.5 us (README.md).
//
// The mix gathers, per chunk of THREADS * N elements, each row's entries in the chunk into a zeroed shared tile (a warp
// per row: binary search on the ascending indices, then a scatter), 8 rows at a time (BEER: 4 rows of both channels),
// and then runs the dense mix's arithmetic on the tiles in the same order: with topk_ratio 1 it is bitwise the
// compressor none.
// The grid is only kTopkCluster CTAs per node, so the step kernels take the registers they need (126-158, no spills)
// rather than a cap that keeps several CTAs resident per SM: with the default cap the fp64 8-deep CHOCO step spilled.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS, 1) choco_topk_step_kernel(const ChocoArgs<T> a) {
  extern __shared__ __align__(16) unsigned char topk_smem[];
  __shared__ TopkShared sh;
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  const int sl = topk_slice(c.n_pad), base = blockIdx.x * sl, len = max(0, min(sl, c.n_pad - base));
  T* sv = reinterpret_cast<T*>(topk_smem);
  unsigned* slive = reinterpret_cast<unsigned*>(sv + sl);
  // theta and x_hat are read before the programmatic-dependency wait, as in choco_step
  bool waited = false;
  for (int j = threadIdx.x * N; j < len; j += THREADS * N) {
    const int i = base + j;
    Pack<T> th = ldv(c.theta + row + i);
    const Pack<T> xh = ldv(a.x_hat + row + i);
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    Pack<T> v;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      th.v[u] -= alpha * g.v[u];
      v.v[u] = th.v[u] - xh.v[u];
    }
    stv(c.theta + row + i, th);
    stv(sv + j, v);
  }
  release_dependents_once(waited);
  topk_live_words(slive, a.live, base, len);
  __syncthreads();
  int pc = 0;
  const TopkThr<T> thr = topk_threshold(sv, len, slive, a.topk_k, sh, pc);
  char* out = code_row(a, ri.par ^ 1, l);
  T* vals = reinterpret_cast<T*>(out);
  unsigned* idx = reinterpret_cast<unsigned*>(out + (size_t)a.topk_k * sizeof(T));
  topk_emit(sv, len, slive, thr, sh, 0, [&](int j, unsigned pos) {
    const T v = sv[j];
    vals[pos] = v;
    idx[pos] = (unsigned)(base + j);
    a.x_hat[row + base + j] += v;
  });
  topk_pad(out, a.topk_k, (int)sizeof(T), a.code_stride);
  cluster_sync();
  end_step(c, l, ri.k, true);
}

template <typename T, int U>
__global__ void __launch_bounds__(THREADS, 1) beer_topk_step_kernel(const BeerArgs<T> a) {
  extern __shared__ __align__(16) unsigned char topk_smem[];
  __shared__ TopkShared sh;
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const size_t row = (size_t)l * c.n_pad;
  const int sl = topk_slice(c.n_pad), base = blockIdx.x * sl, len = max(0, min(sl, c.n_pad - base));
  T* sdx = reinterpret_cast<T*>(topk_smem);       // channel 0: theta - h
  T* sdv = sdx + sl;                               // channel 1: v - g
  unsigned* slive = reinterpret_cast<unsigned*>(sdv + sl);
  // theta, s_g, h, v, g and m_old are read before the programmatic-dependency wait, as in beer_step
  bool waited = false;
  for (int j = threadIdx.x * N; j < len; j += THREADS * N) {
    const int i = base + j;
    const Pack<T> x = ldv(c.theta + row + i), h = ldv(a.h + row + i), g = ldv(a.g + row + i);
    const Pack<T> sg = ldv(a.s_g + row + i), mo = ldv(a.m_old + row + i);
    Pack<T> v = ldv(a.v + row + i);
    release_dependents_once(waited);
    const Pack<T> gr = sum_partials<U>(c, l, i);
    Pack<T> dx, dv;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      v.v[u] += a.gamma * (sg.v[u] - g.v[u]) + gr.v[u] - mo.v[u];
      dx.v[u] = x.v[u] - h.v[u];
      dv.v[u] = v.v[u] - g.v[u];
    }
    stv(a.v + row + i, v);
    stv(a.m_old + row + i, gr);
    stv(sdx + j, dx);
    stv(sdv + j, dv);
  }
  release_dependents_once(waited);
  topk_live_words(slive, a.live, base, len);
  __syncthreads();
  int pc = 0;
#pragma unroll 1
  for (int ch = 0; ch < 2; ++ch) {
    const T* sv = ch == 0 ? sdx : sdv;
    T* est = ch == 0 ? a.h : a.g;
    const TopkThr<T> thr = topk_threshold(sv, len, slive, a.topk_k, sh, pc);
    char* out = beer_code_row(a, ri.par ^ 1, ch, l);
    T* vals = reinterpret_cast<T*>(out);
    unsigned* idx = reinterpret_cast<unsigned*>(out + (size_t)a.topk_k * sizeof(T));
    topk_emit(sv, len, slive, thr, sh, ch, [&](int j, unsigned pos) {
      const T v = sv[j];
      vals[pos] = v;
      idx[pos] = (unsigned)(base + j);
      est[row + base + j] += v;
    });
    topk_pad(out, a.topk_k, (int)sizeof(T), a.code_stride);
  }
  cluster_sync();
  end_step(c, l, ri.k, true);
}

template <typename T>
__global__ void __launch_bounds__(THREADS) choco_topk_mix_kernel(const ChocoArgs<T> a) {
  constexpr int N = Vec<T>::N, CH = THREADS * N, R = THREADS / 32;
  __shared__ __align__(16) T tile[R][CH];
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const char* own = code_row(a, ri.par, l);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, o = threadIdx.x * N;
  Pack<T> zero;
#pragma unroll
  for (int u = 0; u < N; ++u) zero.v[u] = (T)0;
  for (int c0 = blockIdx.x * CH; c0 < c.n_pad; c0 += gridDim.x * CH) {
    Pack<T> t;
    // rows r = 0 (own) .. deg (neighbor r - 1), R at a time: warp q gathers row r0 + q
    for (int r0 = 0; r0 <= deg; r0 += R) {
#pragma unroll
      for (int q = 0; q < R; ++q) stv(&tile[q][o], zero);
      __syncthreads();
      if (r0 + wid <= deg)
        topk_gather(r0 + wid == 0 ? own : nbr_code_row(a, ri.gid, l, r0 + wid - 1, ri.par), a.topk_k, c0, CH, tile[wid], lane);
      __syncthreads();
      for (int q = 0; q < R && r0 + q <= deg; ++q) {
        const Pack<T> d = ldv(&tile[q][o]);
        if (r0 + q == 0) {
          t = d;
#pragma unroll
          for (int u = 0; u < N; ++u) t.v[u] *= ws;
        } else {
          const int e = r0 + q - 1;
#pragma unroll
          for (int u = 0; u < N; ++u) t.v[u] += w[e] * d.v[u];
        }
      }
    }
    const int i = c0 + o;
    if (i < c.n_pad) {
      Pack<T> s = ldv(a.s + row + i);
      const Pack<T> xh = ldv(a.x_hat + row + i);
      Pack<T> th = ldv(c.theta + row + i);
#pragma unroll
      for (int u = 0; u < N; ++u) {
        s.v[u] += t.v[u];
        th.v[u] += a.gamma * (s.v[u] - xh.v[u]);
      }
      stv(a.s + row + i, s);
      stv(c.theta + row + i, th);
    }
    __syncthreads();      // the tiles are read before the next chunk zeroes them
  }
}

template <typename T>
__global__ void __launch_bounds__(THREADS) beer_topk_mix_kernel(const BeerArgs<T> a) {
  constexpr int N = Vec<T>::N, CH = THREADS * N, R = THREADS / 64;
  __shared__ __align__(16) T tile[2][R][CH];
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T alpha = c.alpha[ri.k];
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  // warp wid gathers channel wid / R of row r0 + wid % R
  const int lane = threadIdx.x & 31, ch = (threadIdx.x >> 5) / R, wq = (threadIdx.x >> 5) % R, o = threadIdx.x * N;
  const char* own = beer_code_row(a, ri.par, ch, l);
  Pack<T> zero;
#pragma unroll
  for (int u = 0; u < N; ++u) zero.v[u] = (T)0;
  for (int c0 = blockIdx.x * CH; c0 < c.n_pad; c0 += gridDim.x * CH) {
    Pack<T> th, tg;
    for (int r0 = 0; r0 <= deg; r0 += R) {
#pragma unroll
      for (int q = 0; q < R; ++q) {
        stv(&tile[0][q][o], zero);
        stv(&tile[1][q][o], zero);
      }
      __syncthreads();
      const int r = r0 + wq;
      if (r <= deg)
        topk_gather(r == 0 ? own : reinterpret_cast<const char*>(nbr_row(c, ri.gid, l, r - 1, ri.par, ch)), a.topk_k,
                    c0, CH, tile[ch][wq], lane);
      __syncthreads();
      for (int q = 0; q < R && r0 + q <= deg; ++q) {
        const Pack<T> dh = ldv(&tile[0][q][o]), dg = ldv(&tile[1][q][o]);
        if (r0 + q == 0) {
          th = dh;
          tg = dg;
#pragma unroll
          for (int u = 0; u < N; ++u) {
            th.v[u] *= ws;
            tg.v[u] *= ws;
          }
        } else {
          const T we = w[r0 + q - 1];
#pragma unroll
          for (int u = 0; u < N; ++u) {
            th.v[u] += we * dh.v[u];
            tg.v[u] += we * dg.v[u];
          }
        }
      }
    }
    const int i = c0 + o;
    if (i < c.n_pad) {
      Pack<T> sh = ldv(a.s_h + row + i), sg = ldv(a.s_g + row + i);
      const Pack<T> h = ldv(a.h + row + i), v = ldv(a.v + row + i);
      Pack<T> x = ldv(c.theta + row + i);
#pragma unroll
      for (int u = 0; u < N; ++u) {
        sh.v[u] += th.v[u];
        sg.v[u] += tg.v[u];
        x.v[u] += a.gamma * (sh.v[u] - h.v[u]) - alpha * v.v[u];
      }
      stv(a.s_h + row + i, sh);
      stv(a.s_g + row + i, sg);
      stv(c.theta + row + i, x);
    }
    __syncthreads();
  }
}

// -------------------------------------------------------------------- K-GT ----
// Channel 0 of the published buffer is theta, channel 1 the tracker y (correction mode).  Round k: kgt_mix pulls the
// rows published at the end of round k-1, theta_i <- sum_j W_ij theta_j and c_i += sum_j W_ij y_j - y_i (own terms
// included); then K x [fwd/bwd, kgt_step(p)].  Local DSGD mixes with dsgd_mix_kernel and publishes theta only.
template <typename T>
__global__ void __launch_bounds__(THREADS) kgt_mix_kernel(const KgtArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const T* ys = pub_row(c, ri.par, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> y = ldv(ys + i);
    Pack<T> cr = ldv(a.corr + row + i);
    if (c.sum_mode) {     // W = 11^T / N: theta_i = S_theta / N, c_i += S_y / N - y_i
      const DPack<N> st = network_sum(c, ri.par, 0, i);
      const DPack<N> sy = network_sum(c, ri.par, 1, i);
      Pack<T> th;
#pragma unroll
      for (int u = 0; u < N; ++u) {
        th.v[u] = (T)(st.v[u] / (double)c.n_total);
        cr.v[u] += (T)(sy.v[u] / (double)c.n_total - (double)y.v[u]);
      }
      stv(c.theta + row + i, th);
      stv(a.corr + row + i, cr);
      continue;
    }
    Pack<T> th = ldv(c.theta + row + i), yw;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      th.v[u] *= ws;
      yw.v[u] = ws * y.v[u];
    }
    // for_neighbors<2> written out, as in dsgt_mix: two channels of two neighbors in flight
    for (int e0 = 0; e0 < deg; e0 += 2) {
      Pack<T> qt[2], qy[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          qt[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
          qy[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 1) + i);
        }
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          const T we = w[e0 + j];
#pragma unroll
          for (int u = 0; u < N; ++u) {
            th.v[u] += we * qt[j].v[u];
            yw.v[u] += we * qy[j].v[u];
          }
        }
    }
#pragma unroll
    for (int u = 0; u < N; ++u) cr.v[u] += yw.v[u] - y.v[u];
    stv(c.theta + row + i, th);
    stv(a.corr + row + i, cr);
  }
}

// Local step p of K: u = g + c (CORR; g without it), theta -= alpha_k u, d = u (p = 0) or d + u.  The last step
// publishes theta and y = d / K (one IEEE division, exact for K = 1) into the next parity and ends the round; the
// others keep theta and d local and only advance the draw counters.  Local DSGD writes DSGD's step, th -= alpha * g.
// The 4-deep variant is held to 64 registers (4 CTAs per SM) and the 8-deep one to 128, with no spills: left to the
// compiler, the fp32 IEEE division took the 4-deep correction step to 125 and the fp64 8-deep local step spilled at 80.
template <typename T, int U, bool CORR>
__global__ void __launch_bounds__(THREADS, U <= 4 ? 4 : 2) kgt_step_kernel(const KgtArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const bool first = a.step == 0, last = a.step == a.K - 1;
  const T kf = (T)a.K;
  const size_t row = (size_t)l * c.n_pad;
  // theta, c and d (written by the mix or the previous step, two launches back) are read before the
  // programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    Pack<T> cr, dd;
    if (CORR) {
      cr = ldv(a.corr + row + i);
      if (!first) dd = ldv(a.dacc + row + i);
    }
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    if (CORR) {
#pragma unroll
      for (int u = 0; u < N; ++u) {
        const T uu = g.v[u] + cr.v[u];
        th.v[u] -= alpha * uu;
        dd.v[u] = first ? uu : dd.v[u] + uu;
      }
    } else {
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] -= alpha * g.v[u];
    }
    stv(c.theta + row + i, th);
    if (last) {
      stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
      if (CORR) {
        Pack<T> y;
#pragma unroll
        for (int u = 0; u < N; ++u) y.v[u] = div_rn(dd.v[u], kf);
        stv(pub_row(c, ri.par ^ 1, 1, l) + i, y);
      }
    } else if (CORR) {
      stv(a.dacc + row + i, dd);
    }
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, last);
}

// ------------------------------------------------------------------- DeTAG ----
// Channel 0 of the published buffer is z = theta - alpha y, channel 1 the tracker y.  Gradient round k is K protocol
// rounds p = K k + s, one ag_gossip launch each, then fwd/bwd and detag_track in the last of them.  Sub-step s mixes
// both channels, M_s = sum_j W_ij X_s,j (own term first, then neighbors in table order, as dsgd_mix), and takes
// X_{s+1} = X_{s-1} + w_s (M_s - X_{s-1}); with w_s == 1 it is M_s and X_{s-1} is not read.  X_s is the parity p & 1
// row.  X_{s-1} is the node's own row of parity (p + 1) & 1, which a non-last sub-step overwrites with X_{s+1}: each
// thread reads its element before it writes it, and the round-start wait guarantees the neighbors have finished
// reading it in round p - 1.  The round counter that names the parities was advanced by the previous sub-step, so
// nothing is loaded before the dependency wait.  The last sub-step (LAST) writes theta = X_K and ymix = Y_K, publishes
// nothing and leaves the round open.
template <typename T, bool LAST>
__global__ void __launch_bounds__(THREADS) ag_gossip_kernel(const DetagArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T om = a.omega[a.step];
  const bool acc = om != (T)1;
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const T* xs = pub_row(c, ri.par, 0, l);
  const T* ys = pub_row(c, ri.par, 1, l);
  T* xo = pub_row(c, ri.par ^ 1, 0, l);
  T* yo = pub_row(c, ri.par ^ 1, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> mx = ldv(xs + i), my = ldv(ys + i), px, py;
    if (acc) {
      px = ldv(xo + i);
      py = ldv(yo + i);
    }
#pragma unroll
    for (int u = 0; u < N; ++u) {
      mx.v[u] *= ws;
      my.v[u] *= ws;
    }
    // for_neighbors<2> written out, as in dsgt_mix: two channels of two neighbors in flight
    for (int e0 = 0; e0 < deg; e0 += 2) {
      Pack<T> qx[2], qy[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          qx[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
          qy[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 1) + i);
        }
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          const T we = w[e0 + j];
#pragma unroll
          for (int u = 0; u < N; ++u) {
            mx.v[u] += we * qx[j].v[u];
            my.v[u] += we * qy[j].v[u];
          }
        }
    }
    if (acc) {
#pragma unroll
      for (int u = 0; u < N; ++u) {
        mx.v[u] = px.v[u] + om * (mx.v[u] - px.v[u]);
        my.v[u] = py.v[u] + om * (my.v[u] - py.v[u]);
      }
    }
    if (LAST) {
      stv(c.theta + row + i, mx);
      stv(a.ymix + row + i, my);
    } else {
      stv(xo + i, mx);
      stv(yo + i, my);
    }
  }
  if (!LAST) {
    tag_published(c, l, ri.k);
    finish_round(c, ri.k);
  }
}

// Tracking step of gradient round k, in protocol round p = K k + K - 1: y = Y_K + (g - g_old), g_old = g, and publish
// z = theta - alpha y and y into the other parity.  Y_K (ymix), theta and g_old were written two launches back or
// earlier and are read before the dependency wait; only the gradient partials after it.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) detag_track_kernel(const DetagArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  T* zo = pub_row(c, ri.par ^ 1, 0, l);
  T* yo = pub_row(c, ri.par ^ 1, 1, l);
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> y = ldv(a.ymix + row + i);
    const Pack<T> go = ldv(a.g_old + row + i);
    const Pack<T> th = ldv(c.theta + row + i);
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    Pack<T> z;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      y.v[u] += g.v[u] - go.v[u];
      z.v[u] = th.v[u] - alpha * y.v[u];
    }
    stv(a.g_old + row + i, g);
    stv(zo + i, z);
    stv(yo + i, y);
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ----------------------------------------------------------------- GT-HSGD ----
// dsgt_track with the hybrid estimator in place of the gradient.  g and gp are the sums of the two partial sets (the
// forward/backward at theta and the one at theta_prev, on the same minibatch):
//   v' = g                        in round 0
//      = g + (1 - beta) (v - gp)  otherwise
//   y  = sum_j W_ij y_j + (v' - v);  v <- v';  theta_prev <- theta;  publish theta and y
// Every store is after the pdl_wait.  That matters for theta_prev: the prev-point forward/backward, the launch
// immediately before this one, reads it, and the wait is what orders this write after those reads (the PDL convention
// of common.cuh).  The next round's prev-point launch is three launches later and sees the new row.
template <int U, typename T>
NNDT_DEVINL Pack<T> sum_prev_partials(const HsgdArgs<T>& a, int l, int i) {
  // sum_partials over grad_part_prev: the same issue order and summation order s = 0, 1, 2, ...
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const T* gp = a.grad_part_prev + (size_t)l * c.S * c.n_pad + i;
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

template <typename T, int U>
__global__ void __launch_bounds__(THREADS) hsgd_track_kernel(const HsgdArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const bool first = ri.k == 0;
  const T omb = a.omb;
  const int deg = c.deg[ri.gid * c.L + l];
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const T* ys = pub_row(c, ri.par, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> y;
    if (c.sum_mode) {
      const DPack<N> sy = network_sum(c, ri.par, 1, i);
#pragma unroll
      for (int u = 0; u < N; ++u) y.v[u] = (T)(sy.v[u] / (double)c.n_total);
    } else {
      y = ldv(ys + i);
#pragma unroll
      for (int u = 0; u < N; ++u) y.v[u] *= ws;
      // for_neighbors<4> written out, as in dsgt_track
      for (int e0 = 0; e0 < deg; e0 += 4) {
        Pack<T> q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < deg) q[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 1) + i);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < deg) {
            const T we = w[e0 + j];
#pragma unroll
            for (int u = 0; u < N; ++u) y.v[u] += we * q[j].v[u];
          }
      }
    }
    Pack<T> vn = sum_partials<U>(c, l, i);
    const Pack<T> vo = ldv(a.v + row + i);
    if (!first) {
      const Pack<T> gp = sum_prev_partials<U>(a, l, i);
#pragma unroll
      for (int u = 0; u < N; ++u) vn.v[u] += omb * (vo.v[u] - gp.v[u]);
    }
#pragma unroll
    for (int u = 0; u < N; ++u) y.v[u] += vn.v[u] - vo.v[u];
    const Pack<T> th = ldv(c.theta + row + i);
    stv(a.v + row + i, vn);
    stv(a.theta_prev + row + i, th);
    stv(pub_row(c, ri.par ^ 1, 1, l) + i, y);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
  }
  end_step(c, l, ri.k, true);
}

// --------------------------------------------------------- cross-gradient ----
// Layout and round in consensus.h (XgArgs).  Every neighbor read of protocol round 2k is in xg_pull, after begin_round;
// xg_publish writes only the other parity and ends the protocol round.  Protocol round 2k + 1 is all of xg_step: its
// begin_round waits for the cross-gradients addressed to this node, it pulls them and writes only the other parity.
// Each kernel stores after its pdl_wait: theta_x and xmix are read by the launches of the previous round.
template <typename T>
__global__ void __launch_bounds__(THREADS) xg_pull_kernel(const XgArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const size_t slot = (size_t)c.L * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> own = ldv(c.theta + row + i);
    Pack<T> x = own;
#pragma unroll
    for (int u = 0; u < N; ++u) x.v[u] *= ws;
    // dsgd_mix's accumulation; the same loads are the cross points
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i); },
                     [&](int e, const Pack<T>& q) {
                       stv(a.theta_x + e * slot + row + i, q);
#pragma unroll
                       for (int u = 0; u < N; ++u) x.v[u] += w[e] * q.v[u];
                     });
    // an idle slot computes a finite gradient at the own row, never published
    for (int e = deg; e < c.dmax; ++e) stv(a.theta_x + e * slot + row + i, own);
    stv(a.xmix + row + i, x);
  }
}

// the own gradient into g, and slot e's gradient into channel 1 + e of the other parity for e < deg; every sum in the
// order s = 0, 1, 2, ... (sum_partials, as hsgd_track sums both of its sets)
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) xg_publish_kernel(const XgArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  const size_t row = (size_t)l * c.n_pad;
  const size_t slot = (size_t)c.L * c.S * c.n_pad;
  const T* gx = a.grad_part_x + (size_t)l * c.S * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    for (int e = 0; e < deg; ++e)
      stv(pub_row(c, ri.par ^ 1, 1 + e, l) + i, sum_partial_rows<U>(gx + e * slot + i, c.S, c.n_pad));
    stv(a.g + row + i, sum_partials<U>(c, l, i));
  }
  tag_published(c, l, ri.k);
  finish_round(c, ri.k);
}

// d = coef0 g + sum_e coef_e g_{j_e -> i} in fp64, own term first and then table order, rounded once to T; then
// dsgd_step's arithmetic on (xmix, d)
template <typename T>
__global__ void __launch_bounds__(THREADS) xg_step_kernel(const XgArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T alpha = c.alpha[ri.k];
  const double c0 = a.coef0[ri.gid * c.L + l];
  const double* ce = a.coef + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> g = ldv(a.g + row + i);
    DPack<N> d;
#pragma unroll
    for (int u = 0; u < N; ++u) d.v[u] = c0 * (double)g.v[u];
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 1 + e) + i); },
                     [&](int e, const Pack<T>& q) {
                       const double we = ce[e];
#pragma unroll
                       for (int u = 0; u < N; ++u) d.v[u] += we * (double)q.v[u];
                     });
    Pack<T> dt, th = ldv(a.xmix + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) dt.v[u] = (T)d.v[u];
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] -= alpha * dt.v[u];
    stv(c.theta + row + i, th);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
  }
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------- Gossip-PGA ----
// Round k: pga_sum, pga_mix, fwd/bwd, dsgd_step (DSGD's, unchanged).  Global round (k mod period == period - 1):
// pga_sum reduces this rank's published rows of round k into its fp64 partial, as local_sum_kernel does, and posts the
// sum flag k + 1; pga_mix waits for every rank's partial and writes the network mean into theta, as dsgd_mix_kernel's
// complete-graph mode does.  Gossip round: pga_sum returns at once and pga_mix is dsgd_mix_kernel's pointer-table mix
// (gossip) or leaves theta as it is (local SGD).
// pga_sum's grid is one CTA per THREADS vectors of the row, far from filling the SMs, so it asks for one resident CTA
// per SM: with the default bound the fp64 variant spilled 4 bytes (96 registers without the bound's pressure).
template <typename T>
__global__ void __launch_bounds__(THREADS, 1) pga_sum_kernel(const PgaArgs<T> a) {
  const Common<T>& c = a.c;
  pdl_wait();
  pdl_launch_dependents();
  const RoundInfo<T> ri = round_info(c);
  const PgaPhase ph = pga_phase(ri.k, a.period);
  if (!ph.global) return;
  constexpr int N = Vec<T>::N;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    double s[N];
#pragma unroll
    for (int u = 0; u < N; ++u) s[u] = 0.0;
    for (int l = 0; l < c.L; ++l) {
      const Pack<T> q = ldv(pub_row(c, ri.par, 0, l) + i);
#pragma unroll
      for (int u = 0; u < N; ++u) s[u] += (double)q.v[u];
    }
    double* dst = c.sum_local + (size_t)(ph.sum_par * c.C) * c.n_pad + i;
#pragma unroll
    for (int u = 0; u < N; u += 2) *reinterpret_cast<double2*>(dst + u) = make_double2(s[u], s[u + 1]);
  }
  // last block: tell every peer that this rank's partial sum of round k is ready
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(c.done_ctr, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last) {
    if (threadIdx.x == 0) *c.done_ctr = 0;
    if (c.world > 1) {
      __threadfence_system();
      if ((int)threadIdx.x < c.world && (int)threadIdx.x != c.rank)
        st_release_sys(reinterpret_cast<int*>(c.peer_sum_flag[threadIdx.x]), ri.k + 1);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(THREADS) pga_mix_kernel(const PgaArgs<T> a) {
  const Common<T>& c = a.c;
  pdl_wait();
  pdl_launch_dependents();
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const size_t row = (size_t)l * c.n_pad;
  const PgaPhase ph = pga_phase(ri.k, a.period);
  if (ph.global) {     // theta_i <- the network mean of the rows published for round k
    if (c.world > 1 && blockIdx.x == 0 && blockIdx.y == 0) announce_round(c, ri.k);
    wait_all_sums(c, ri.k);
    for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
      const DPack<N> sall = network_sum(c, ph.sum_par, 0, i);
      Pack<T> th;
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] = (T)(sall.v[u] / (double)c.n_total);
      stv(c.theta + row + i, th);
    }
    return;
  }
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);      // c.sum_mode is 0: the neighbor wait (none on the edgeless graph of local SGD)
  if (!a.gossip) return;
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] *= ws;
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i); },
                     [&](int e, const Pack<T>& q) {
#pragma unroll
                       for (int u = 0; u < N; ++u) th.v[u] += w[e] * q.v[u];
                     });
    stv(c.theta + row + i, th);
  }
}

// ----------------------------------------------------------------- SlowMo ----
// Round k: pga_sum, pga_mix, slowmo_outer, fwd/bwd, dsgd_step or dsgdm_step (both unchanged).  A separate launch keeps
// pga_mix as Gossip-PGA has it.  On a global round, after pga_mix wrote xbar into theta (consensus.h: SlowmoArgs):
//   u <- beta_s u + (a - xbar) / gamma;  a <- a - (alpha_s gamma) u;  theta <- a;  m <- 0
// in fp64 from the stored rows, every operation rounded on its own (no contraction, as the PyTorch path computes it),
// each stored row rounded once.  A zeroed m makes the next dsgdm_step take its round-0 step.  Every store is after the
// pdl_wait: theta is pga_mix's, m the previous round's step's.
template <typename T>
__global__ void __launch_bounds__(THREADS) slowmo_outer_kernel(const SlowmoArgs<T> a) {
  const Common<T>& c = a.c;
  pdl_wait();
  pdl_launch_dependents();
  const RoundInfo<T> ri = round_info(c);
  if (!pga_phase(ri.k, a.period).global) return;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const size_t row = (size_t)l * c.n_pad;
  const double gamma = ri.k == 0 ? (double)a.alpha0 : (double)c.alpha[ri.k - 1];
  const double step = __dmul_rn(a.slow_lr, gamma);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> x = ldv(c.theta + row + i);
    Pack<T> an = ldv(a.anchor + row + i), uu = ldv(a.u + row + i);
#pragma unroll
    for (int v = 0; v < N; ++v) {
      const double un = __dadd_rn(__dmul_rn(a.slow_momentum, (double)uu.v[v]),
                                  div_rn(__dsub_rn((double)an.v[v], (double)x.v[v]), gamma));
      uu.v[v] = (T)un;
      an.v[v] = (T)__dsub_rn((double)an.v[v], __dmul_rn(step, un));
    }
    stv(a.u + row + i, uu);
    stv(a.anchor + row + i, an);
    stv(c.theta + row + i, an);
    if (a.m != nullptr) {
      Pack<T> z;
#pragma unroll
      for (int v = 0; v < N; ++v) z.v[v] = (T)0;
      stv(a.m + row + i, z);
    }
  }
}

// ---------------------------------------------------------------- DP-DSGD ----
// Round k (stream and rules in consensus.h: DpArgs): dsgd_mix, fwd/bwd, dp_norm, dp_step.  The clip factor needs the
// norm of the whole gradient row, which is spread over the CTAs of the node, so the norm takes a launch of its own:
// dp_norm sums the partials as the step will and writes one fp64 partial of sum g^2 per fixed chunk of the row (the
// partials do not depend on the one-wave grid, as cg_dist's), dp_step adds them in chunk order.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) dp_norm_kernel(const DpArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nchunk = cg_chunks(c);
  __shared__ double red[THREADS / 32];
  for (int ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
    const int i = (ch * THREADS + threadIdx.x) * N;
    double s = 0.0;
    if (i < c.n_pad) {
      const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
      for (int u = 0; u < N; ++u) s += (double)g.v[u] * (double)g.v[u];
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = red[0];
#pragma unroll
      for (int w = 1; w < THREADS / 32; ++w) t += red[w];
      a.norm_part[(size_t)l * a.pstride + ch] = t;
    }
    __syncthreads();
  }
}

// theta_i -= alpha_k (f_i g_i + v_i) and publish.  With no noise the step is f_i g_i rounded on its own, so f_i = 1 is
// dsgd_step's arithmetic bit for bit.
template <typename T, int U>
__global__ void __launch_bounds__(THREADS) dp_step_kernel(const DpArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const size_t row = (size_t)l * c.n_pad;
  const int i0 = (blockIdx.x * THREADS + threadIdx.x) * N;
  // theta was last written by dsgd_mix, three launches back: the first vector is loaded before the dependency wait
  Pack<T> th0;
  if (i0 < c.n_pad) th0 = ldv(c.theta + row + i0);
  pdl_wait();
  pdl_launch_dependents();
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  __shared__ double fsh;
  if (threadIdx.x == 0) {
    const double* np = a.norm_part + (size_t)l * a.pstride;
    const int nchunk = cg_chunks(c);
    double s = 0.0;
    for (int ch = 0; ch < nchunk; ++ch) s += np[ch];
    const double nrm = sqrt(s);
    fsh = nrm > a.clip ? a.clip / nrm : 1.0;
  }
  __syncthreads();
  const T f = (T)fsh;
  const bool noisy = a.cz_dp != 0.0 || a.cz_pair != 0.0;
  const int deg = c.deg[ri.gid * c.L + l];
  const int* ids = a.nbr_id + (size_t)(ri.gid * c.L + l) * c.dmax;
  const unsigned me = (unsigned)(a.node0 + l);
  for (int i = i0; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = i == i0 ? th0 : ldv(c.theta + row + i);
    const Pack<T> g = sum_partials<U>(c, l, i);
    Pack<T> u;
#pragma unroll
    for (int q = 0; q < N; ++q) u.v[q] = mul_rn(f, g.v[q]);
    if (noisy) {
      const Pack<T> v = dp_noise(a, ri.k, me, deg, ids, i);
#pragma unroll
      for (int q = 0; q < N; ++q) u.v[q] += v.v[q];
    }
#pragma unroll
    for (int q = 0; q < N; ++q) th.v[q] -= alpha * u.v[q];
    stv(c.theta + row + i, th);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
  }
  end_step(c, l, ri.k, true);
}

// ---------------------------------------------------------------- Moniqua ----
// Round k (layout, stream and rules in consensus.h: MoniquaArgs): mq_mix, fwd/bwd, mq_step.  mq_mix pulls one 32-bit
// code word per neighbor and thread (the codes of its Vec<T>::N elements), decodes in registers against y = theta_i
// (y / B once per element) and accumulates sum_{j != i} w_ij (xhat_j - xhat_i) in fp64 in neighbor order, each product
// rounded on its own, so the host twin computes the same bits.  The margin hits of a warp go out in one atomic.
template <typename T, int BITS>
__global__ void __launch_bounds__(THREADS) mq_mix_kernel(const MoniquaArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  constexpr unsigned MASK = (1u << BITS) - 1u;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const unsigned* own = mq_code_row(a, ri.par, l);
  const double lim = 0.5 - 1.0 / (1 << BITS);
  unsigned hits = 0u;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    const unsigned cw = mq_word<T, BITS>(own, i);
    double yb[N], xi[N], acc[N];
#pragma unroll
    for (int u = 0; u < N; ++u) {
      double off;
      yb[u] = __ddiv_rn((double)th.v[u], a.B);
      xi[u] = mq_decode<BITS>((cw >> (u * BITS)) & MASK, yb[u], a.B, off);
      acc[u] = 0.0;
    }
    for_neighbors<4>(deg, [&](int e) { return mq_word<T, BITS>(reinterpret_cast<const unsigned*>(nbr_row(c, ri.gid, l, e, ri.par, 0)), i); },
                     [&](int e, unsigned q) {
                       const double we = (double)w[e];
#pragma unroll
                       for (int u = 0; u < N; ++u) {
                         double off;
                         const double xj = mq_decode<BITS>((q >> (u * BITS)) & MASK, yb[u], a.B, off);
                         acc[u] = __dadd_rn(acc[u], __dmul_rn(we, __dsub_rn(xj, xi[u])));
                         hits += fabs(off) > lim ? 1u : 0u;
                       }
                     });
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] = (T)__dadd_rn((double)th.v[u], acc[u]);
    stv(c.theta + row + i, th);
  }
  hits = __reduce_add_sync(0xffffffffu, hits);
  if ((threadIdx.x & 31) == 0 && hits != 0u) atomicAdd(a.margin + l, (unsigned long long)hits);
}

// DSGD's step (ED = false) or ed_step's adapt / correct (ED: psi <- theta in round 0), then the code of the new theta
// for round k + 1.  The loop runs per warp, as choco_step: the G lanes holding one code word OR their bits together with
// xor shuffles and the first of them stores the word; a lane past the end of the row takes part and stores nothing.
template <typename T, int U, int BITS, bool ED>
__global__ void __launch_bounds__(THREADS) mq_step_kernel(const MoniquaArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  constexpr int G = 32 / BITS / N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const bool init = ri.k == 0;
  const size_t row = (size_t)l * c.n_pad;
  unsigned* out = mq_code_row(a, ri.par ^ 1, l);
  const unsigned me = (unsigned)(a.node0 + l);
  const int lane = threadIdx.x & 31;
  // theta (written by the mix two launches back) and psi (the previous round's step) are read before the
  // programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int w0 = (blockIdx.x * THREADS + (threadIdx.x & ~31)) * N; w0 < c.n_pad; w0 += gridDim.x * THREADS * N) {
    const int i = w0 + lane * N;
    const bool in = i < c.n_pad;
    Pack<T> th, dc;
#pragma unroll
    for (int u = 0; u < N; ++u) { th.v[u] = (T)0; dc.v[u] = (T)0; }
    if (in) {
      th = ldv(c.theta + row + i);
      if (ED && !init) {
        const Pack<T> ps = ldv(a.psi + row + i);
#pragma unroll
        for (int u = 0; u < N; ++u) dc.v[u] = th.v[u] - ps.v[u];
      }
    }
    release_dependents_once(waited);
    unsigned bits = 0u;
    if (in) {
      const Pack<T> g = sum_partials<U>(c, l, i);
      if (ED) {
        Pack<T> pn;
#pragma unroll
        for (int u = 0; u < N; ++u) {
          pn.v[u] = th.v[u] - alpha * g.v[u];
          th.v[u] = pn.v[u] + dc.v[u];
        }
        stv(a.psi + row + i, pn);
      } else {
#pragma unroll
        for (int u = 0; u < N; ++u) th.v[u] -= alpha * g.v[u];
      }
      stv(c.theta + row + i, th);
      const uint4 r = curand_Philox4x32_10(make_uint4((unsigned)(i >> 2), (unsigned)(ri.k + 1), me, kMqTag),
                                           make_uint2(a.key0, a.key1));
      const unsigned lw = a.live[i >> 5];
#pragma unroll
      for (int u = 0; u < N; ++u) {
        const int q = (i & 3) + u;
        const unsigned rr = q == 0 ? r.x : q == 1 ? r.y : q == 2 ? r.z : r.w;
        const unsigned code = ((lw >> ((i & 31) + u)) & 1u) ? mq_code<BITS>((double)th.v[u], a.B, rr) : 0u;
        bits |= code << (((i + u) * BITS) & 31);
      }
    }
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) bits |= __shfl_xor_sync(0xffffffffu, bits, o);
    if (in && (lane & (G - 1)) == 0) out[(i * BITS) >> 5] = bits;
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ---------------------------------------------------------------- SPARQ-SGD ----
// Round k (layout and rules in consensus.h: SparqArgs): sparq_mix, H x [fwd/bwd, sparq_step(p)], sparq_publish.
// sparq_mix reads the tails of the node's own row and of its neighbors' rows of parity k & 1 after the round-start wait,
// lists the triggered neighbor slots in table order (one warp ballot per 32 slots; a node has at most THREADS
// neighbors, ops/engine.py: check_wait_capacity) and runs choco_mix's arithmetic over the own row, when triggered, and
// the listed slots only: a row whose tail says 0 is never read past its tail.  With a zero code choco_mix would add
// W_ij * 0 for it, so with every code of a non-triggered node zero (threshold 0) the mix is choco_mix bit for bit.
template <typename T, int Q>
__global__ void __launch_bounds__(THREADS) sparq_mix_kernel(const SparqArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  __shared__ int slot[THREADS];
  __shared__ unsigned wmask[THREADS / 32];
  __shared__ int own_trig;
  const char* own = sparq_row(a, ri.par, l);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int e = threadIdx.x;
  const bool f = e < deg && sparq_trig(reinterpret_cast<const char*>(nbr_row(c, ri.gid, l, e, ri.par, 0)), a.code_bytes);
  const unsigned m = __ballot_sync(0xffffffffu, f);
  if (lane == 0) wmask[warp] = m;
  if (threadIdx.x == 0) own_trig = sparq_trig(own, a.code_bytes);
  __syncthreads();
  int before = 0, nsel = 0;
#pragma unroll
  for (int q = 0; q < THREADS / 32; ++q) {
    const int cnt = __popc(wmask[q]);
    before += q < warp ? cnt : 0;
    nsel += cnt;
  }
  if (f) slot[before + __popc(m & ((1u << lane) - 1u))] = e;
  __syncthreads();
  const bool ot = own_trig != 0;
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const unsigned lw = Q == kCodeSign ? a.live[i >> 5] : 0u;
    Pack<T> t;
    if (ot) {
      t = choco_decode<T, Q>(own, c.n_pad, i, lw);
#pragma unroll
      for (int u = 0; u < N; ++u) t.v[u] *= ws;
    } else {
#pragma unroll
      for (int u = 0; u < N; ++u) t.v[u] = (T)0;
    }
    for_neighbors<4>(nsel, [&](int j) {
                       return choco_decode<T, Q>(reinterpret_cast<const char*>(nbr_row(c, ri.gid, l, slot[j], ri.par, 0)),
                                                 c.n_pad, i, lw);
                     },
                     [&](int j, const Pack<T>& q) {
                       const T we = w[slot[j]];
#pragma unroll
                       for (int u = 0; u < N; ++u) t.v[u] += we * q.v[u];
                     });
    Pack<T> s = ldv(a.s + row + i);
    const Pack<T> xh = ldv(a.x_hat + row + i);
    Pack<T> th = ldv(c.theta + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) {
      s.v[u] += t.v[u];
      th.v[u] += a.gamma * (s.v[u] - xh.v[u]);
    }
    stv(a.s + row + i, s);
    stv(c.theta + row + i, th);
  }
}

// Local step p of H: theta -= alpha_k g (dsgd_step's expression).  The loop walks dp_norm's chunks (chunk ch is the
// grid-stride iteration that covers it), so the last step writes one fp64 partial of sum (theta - x_hat)^2 per chunk,
// reduced as dp_norm reduces: in element order per thread, xor shuffles per warp, warps in order.  The partials do not
// depend on the grid, the local node count or the launch order.  Steps p < H - 1 end as K-GT's do; the last one leaves
// the draw counter and the round to sparq_publish, which ends the round without drawing again (H draws per round).
// As kgt_step, the 4-deep variant is held to 64 registers and the 8-deep one to 128: left to the compiler, the 8-deep
// steps spilled at 64.
template <typename T, int U, bool LAST>
__global__ void __launch_bounds__(THREADS, U <= 4 ? 4 : 2) sparq_step_kernel(const SparqArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  const int nchunk = cg_chunks(c);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ double red[THREADS / 32];
  // theta (the mix or the previous step, two launches back) and x_hat (the previous round's publish) are read before
  // the programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
    const int i = (ch * THREADS + threadIdx.x) * N;
    double sq = 0.0;
    if (i < c.n_pad) {
      Pack<T> th = ldv(c.theta + row + i);
      Pack<T> xh;
      if (LAST) xh = ldv(a.x_hat + row + i);
      release_dependents_once(waited);
      const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
      for (int u = 0; u < N; ++u) th.v[u] -= alpha * g.v[u];
      stv(c.theta + row + i, th);
      if (LAST) {
#pragma unroll
        for (int u = 0; u < N; ++u) {
          const T d = th.v[u] - xh.v[u];
          sq += (double)d * (double)d;
        }
      }
    }
    if (LAST) {
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      if (lane == 0) red[warp] = sq;
      __syncthreads();
      if (threadIdx.x == 0) {
        double t = red[0];
#pragma unroll
        for (int q = 1; q < THREADS / 32; ++q) t += red[q];
        a.norm_part[(size_t)l * a.pstride + ch] = t;
      }
      __syncthreads();
    }
  }
  release_dependents_once(waited);
  if (!LAST) end_step(c, l, ri.k, false);
}

// e_i = the partials in chunk order (thread 0, into shared memory: every CTA of the node takes the same decision) and
// trig = e_i > thr[k].  On a trigger the code of v = theta - x_hat goes into parity (k+1) & 1 with choco_encode and
// x_hat += dec; a non-triggered node writes no code byte.  CTA 0 of the node writes the tail and counts the trigger.
template <typename T, int Q>
__global__ void __launch_bounds__(THREADS) sparq_publish_kernel(const SparqArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  __shared__ double esh;
  if (threadIdx.x == 0) {
    const double* np = a.norm_part + (size_t)l * a.pstride;
    const int nchunk = cg_chunks(c);
    double s = 0.0;
    for (int ch = 0; ch < nchunk; ++ch) s += np[ch];
    esh = s;
  }
  __syncthreads();
  const double e = esh;
  const bool trig = e > a.thr[ri.k];
  char* out = sparq_row(a, ri.par ^ 1, l);
  const size_t row = (size_t)l * c.n_pad;
  const int lane = threadIdx.x & 31;
  if (trig) {
    for (int w0 = (blockIdx.x * THREADS + (threadIdx.x & ~31)) * N; w0 < c.n_pad; w0 += gridDim.x * THREADS * N) {
      const int i = w0 + lane * N;
      const bool in = i < c.n_pad;
      Pack<T> th, xh, v;
#pragma unroll
      for (int u = 0; u < N; ++u) { th.v[u] = (T)0; xh.v[u] = (T)0; }
      if (in) {
        th = ldv(c.theta + row + i);
        xh = ldv(a.x_hat + row + i);
      }
#pragma unroll
      for (int u = 0; u < N; ++u) v.v[u] = th.v[u] - xh.v[u];
      const Pack<T> d = choco_encode<T, Q>(v, out, c.n_pad, i, in, lane, a.live);
      if (in) {
#pragma unroll
        for (int u = 0; u < N; ++u) xh.v[u] += d.v[u];
        stv(a.x_hat + row + i, xh);
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned* tail = reinterpret_cast<unsigned*>(out + a.code_bytes);
    tail[0] = trig ? 1u : 0u;
    tail[1] = 0u;
    *reinterpret_cast<double*>(out + a.code_bytes + 8) = e;
    a.triggers[l] += trig ? 1 : 0;
  }
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------- decentralized AMSGrad / AdaGrad ----
// Channel 0 of the published buffer is theta, channel 1 the second-moment tracker u~ (tracking).  Round k:
// dadaptive_mix pulls the rows published at the end of round k-1, x_i = sum_j W_ij theta_j into theta and
// z_i = sum_j W_ij u~_j into ut (own terms included: the own u~ is the node's published row, since ut holds z); then
// fwd/bwd and dadaptive_step.  Without tracking the mix is dsgd_mix_kernel.
template <typename T>
__global__ void __launch_bounds__(THREADS) dadaptive_mix_kernel(const DAdaptiveArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const size_t row = (size_t)l * c.n_pad;
  const T* us = pub_row(c, ri.par, 1, l);
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th, z;
    if (c.sum_mode) {     // W = 11^T / N: x_i = S_theta / N, z_i = S_u~ / N
      const DPack<N> st = network_sum(c, ri.par, 0, i);
      const DPack<N> su = network_sum(c, ri.par, 1, i);
#pragma unroll
      for (int u = 0; u < N; ++u) {
        th.v[u] = (T)(st.v[u] / (double)c.n_total);
        z.v[u] = (T)(su.v[u] / (double)c.n_total);
      }
      stv(c.theta + row + i, th);
      stv(a.ut + row + i, z);
      continue;
    }
    th = ldv(c.theta + row + i);
    z = ldv(us + i);
#pragma unroll
    for (int u = 0; u < N; ++u) {
      th.v[u] *= ws;
      z.v[u] *= ws;
    }
    // for_neighbors<2> written out, as in dsgt_mix: two channels of two neighbors in flight
    for (int e0 = 0; e0 < deg; e0 += 2) {
      Pack<T> qt[2], qu[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          qt[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
          qu[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 1) + i);
        }
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (e0 + j < deg) {
          const T we = w[e0 + j];
#pragma unroll
          for (int u = 0; u < N; ++u) {
            th.v[u] += we * qt[j].v[u];
            z.v[u] += we * qu[j].v[u];
          }
        }
    }
    stv(c.theta + row + i, th);
    stv(a.ut + row + i, z);
  }
}

// The step on the mixed row x (theta after the mix), with alpha_k from the schedule:
//   m <- beta1 m + (1 - beta1) g
//   amsgrad (!ADAGRAD):  v <- beta2 v + (1 - beta2) g^2;  vhat' = max(vhat, v)
//   adagrad:             vhat' = vhat + (g^2 - vhat) / (k + 1)        (k from the round counter: right after a resume)
//   TRACK:  u~ = z + (vhat' - vhat), u = max(u~, eps);   otherwise u = max(vhat', eps)
//   theta <- x - alpha_k m / sqrt(u);  m, v and vhat' are stored, theta (and u~) published into the next parity.
// u~ is not stored: the next mix reads the node's own published row.  The square root and the quotients are correctly
// rounded (sqrt_rn / div_rn), so the fp32 step carries a few units of round-off, not the approximations of
// --use_fast_math.  The 4-deep variant is held to 80 registers (3 CTAs per SM) and the 8-deep one to 128, with no
// spills: at kgt_step's 64 the fp64 steps and the fp32 tracked AMSGrad step spilled around the IEEE slow paths.
template <typename T, int U, bool ADAGRAD, bool TRACK>
__global__ void __launch_bounds__(THREADS, U <= 4 ? 3 : 2) dadaptive_step_kernel(const DAdaptiveArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const T b1 = a.beta1, b1c = (T)1 - a.beta1, b2 = a.beta2, b2c = (T)1 - a.beta2, eps = a.eps;
  const T cnt = (T)(ri.k + 1);
  const size_t row = (size_t)l * c.n_pad;
  // theta and z (written by the mix two launches back) and m, v, vhat (the previous round's step) are read before the
  // programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    Pack<T> m = ldv(a.m + row + i);
    Pack<T> vh = ldv(a.vhat + row + i);
    Pack<T> v, z;
    if (!ADAGRAD) v = ldv(a.v + row + i);
    if (TRACK) z = ldv(a.ut + row + i);
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
    for (int u = 0; u < N; ++u) {
      m.v[u] = b1 * m.v[u] + b1c * g.v[u];
      const T g2 = g.v[u] * g.v[u];
      T vn;
      if (ADAGRAD) {
        vn = vh.v[u] + div_rn(g2 - vh.v[u], cnt);
      } else {
        v.v[u] = b2 * v.v[u] + b2c * g2;
        vn = v.v[u] > vh.v[u] ? v.v[u] : vh.v[u];
      }
      T uu;
      if (TRACK) {
        z.v[u] += vn - vh.v[u];             // u~
        uu = z.v[u] > eps ? z.v[u] : eps;
      } else {
        uu = vn > eps ? vn : eps;
      }
      vh.v[u] = vn;
      th.v[u] -= alpha * div_rn(m.v[u], sqrt_rn(uu));
    }
    stv(a.m + row + i, m);
    if (!ADAGRAD) stv(a.v + row + i, v);
    stv(a.vhat + row + i, vh);
    stv(c.theta + row + i, th);
    stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
    if (TRACK) stv(pub_row(c, ri.par ^ 1, 1, l) + i, z);
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ---------------------------------------------------------------- RelaySum ----
// Layout in consensus.h.  Round k: relay_mix pulls the deg messages published for this node at the end of round k-1
// (r_e = m_{j_e -> l}, e ascending), keeps them in rin and writes x = h + (sum_e r_e - (R_l^k - 1) h) / n into theta;
// then fwd/bwd and relay_step.  The product and the quotient are rounded on their own (mul_rn / div_rn), as the PyTorch
// ops round them.  Every neighbor read of the round is in this kernel.
template <typename T>
__global__ void __launch_bounds__(THREADS) relay_mix_kernel(const RelayArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T rm1 = a.reach[l * (a.diam + 1) + min(ri.k, a.diam)];
  const size_t row = (size_t)l * c.n_pad;
  T* rin = a.rin + (size_t)l * c.dmax * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> x = ldv(c.theta + row + i), s;
#pragma unroll
    for (int u = 0; u < N; ++u) s.v[u] = (T)0;
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i); },
                     [&](int e, const Pack<T>& q) {
                       stv(rin + (size_t)e * c.n_pad + i, q);
#pragma unroll
                       for (int u = 0; u < N; ++u) s.v[u] += q.v[u];
                     });
#pragma unroll
    for (int u = 0; u < N; ++u) x.v[u] += div_rn(s.v[u] - mul_rn(rm1, x.v[u]), a.n);
    stv(c.theta + row + i, x);
  }
}

// h = x - alpha_k g into theta, and for each neighbor e the message h + sum_{e' != e} r_e' (e' ascending) into channel e
// of parity k+1.  theta and the D received rows (written by the mix two launches back) are read before the
// programmatic-dependency wait, the gradient partials after it.  A star hub of degree deg adds deg (deg - 1) rows per
// element.  -Xptxas -v, no spills: <T, 4, 4> is held to 80 registers (3 CTAs per SM), <T, 8, 4> and <T, 4, 16> to
// 128 (2 CTAs).  <T, 8, 16> spilled at 128, so a node of degree above 4 sums its partials 4 deep.
template <typename T, int U, int D>
__global__ void __launch_bounds__(THREADS, U <= 4 && D <= 4 ? 3 : 2) relay_step_kernel(const RelayArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  const T* rin = a.rin + (size_t)l * c.dmax * c.n_pad;
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> h = ldv(c.theta + row + i);
    Pack<T> r[D];
    // the D received rows are prefetched with theta while the partials fit beside them (U = 4 with D = 4); otherwise
    // they are loaded after the partials are summed, whose registers are then free
    constexpr bool kPrefetch = U <= 4 && D <= 4;
    if (kPrefetch) {
#pragma unroll
      for (int e = 0; e < D; ++e)
        if (e < deg) r[e] = ldv(rin + (size_t)e * c.n_pad + i);
    }
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    if (!kPrefetch) {
#pragma unroll
      for (int e = 0; e < D; ++e)
        if (e < deg) r[e] = ldv(rin + (size_t)e * c.n_pad + i);
    }
#pragma unroll
    for (int u = 0; u < N; ++u) h.v[u] -= alpha * g.v[u];
    stv(c.theta + row + i, h);
#pragma unroll
    for (int e = 0; e < D; ++e)
      if (e < deg) {
        Pack<T> m = h;
#pragma unroll
        for (int f = 0; f < D; ++f)
          if (f < deg && f != e) {
#pragma unroll
            for (int u = 0; u < N; ++u) m.v[u] += r[f].v[u];
          }
        stv(pub_row(c, ri.par ^ 1, e, l) + i, m);
      }
  }
  release_dependents_once(waited);
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------- PowerGossip ----
// Layout in consensus.h.  Round k runs phase k & 1: pg_mix, fwd/bwd, pg_step.  Every neighbor read of the round is in
// pg_mix, after begin_round; pg_step writes only the other parity.
template <typename T>
NNDT_DEVINL T* pg_row(const PgArgs<T>& a, int par, int chan, int l) {
  const Common<T>& c = a.c;
  return c.pub + ((size_t)(par * c.C + chan) * c.pub_L + l) * a.W;
}

// Each CTA of node l pulls the deg messages of round k (own channel e and the one neighbor j_e wrote for l, 4 elements
// in flight per thread) into shared memory as d_e = a_lo - a_hi: the same bits at both endpoints.  CTA 0 then writes
// the next vectors d / |d|, one warp per (edge, matrix): |d|^2 is summed in fp64 by the lanes in element order and
// combined by xor butterflies, an order that depends on nothing but the difference (ops/consensus_ref.py: pg_sumsq), so
// both endpoints store the same bits; a zero difference keeps the stored vector.  Phase 0 writes p and reads q, phase 1
// writes q and reads p, so the other CTAs never read what CTA 0 writes.  Every CTA applies
// x = h - gamma sum_e (W_ie s_ie) U_e to its grid-stride share of the row.
template <typename T>
__global__ void __launch_bounds__(THREADS) pg_mix_kernel(const PgArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  extern __shared__ __align__(16) unsigned char pg_smem[];
  T* d = reinterpret_cast<T*>(pg_smem);                 // [deg, W] canonical differences
  __shared__ T coef[kPgMaxDeg];                         // W_ie s_ie
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const int ph = ri.par;
  const int len = (ph ? a.Q : a.P) + a.B;
  const int* sg = a.sign + l * c.dmax;
  if ((int)threadIdx.x < deg) coef[threadIdx.x] = c.nbr_w[(ri.gid * c.L + l) * c.dmax + threadIdx.x] * (T)sg[threadIdx.x];
  const int total = deg * len;
  for (int b = threadIdx.x; b < total; b += 4 * THREADS) {
    T own[4], nb[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = b + u * THREADS;
      if (t < total) {
        const int e = t / len, j = t - e * len;
        own[u] = pg_row(a, ph, e, l)[j];
        nb[u] = nbr_row(c, ri.gid, l, e, ph, 0)[j];
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = b + u * THREADS;
      if (t < total) {
        const int e = t / len, j = t - e * len;
        d[e * a.W + j] = sg[e] > 0 ? own[u] - nb[u] : nb[u] - own[u];
      }
    }
  }
  __syncthreads();
  const int PQ = a.P + a.Q;
  T* vl = a.vec + (size_t)l * c.dmax * PQ;
  if (blockIdx.x == 0) {
    const int lane = threadIdx.x & 31;
    for (int t = threadIdx.x >> 5; t < deg * a.nseg; t += THREADS / 32) {
      const int e = t / a.nseg;
      const int* sd = a.seg + 5 * (t - e * a.nseg);
      if (sd[2] == 0) continue;                          // a 1-D tensor has no vectors
      const int ln = ph ? sd[2] : sd[1];
      const T* dv = d + e * a.W + (ph ? sd[4] : sd[3]);
      double ss = 0.0;
      for (int j = lane; j < ln; j += 32) {
        const double x = (double)dv[j];
        ss = __dadd_rn(ss, __dmul_rn(x, x));
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) ss = __dadd_rn(ss, __shfl_xor_sync(0xffffffffu, ss, o));
      if (ss > 0.0) {
        const double nrm = sqrt_rn(ss);
        T* out = vl + (size_t)e * PQ + (ph ? a.P + sd[4] : sd[3]);
        for (int j = lane; j < ln; j += 32) out[j] = (T)div_rn((double)dv[j], nrm);
      }
    }
  }
  T* th = c.theta + (size_t)l * c.n_pad;
  const int gt = blockIdx.x * THREADS + threadIdx.x, gs = gridDim.x * THREADS;
  const int base = ph ? a.Q : a.P;
  for (int s = 0; s < a.nseg; ++s) {
    const int* sd = a.seg + 5 * s;
    const int off = sd[0], m = sd[1], n = sd[2], poff = sd[3], qoff = sd[4];
    const int numel = n > 0 ? m * n : m;
    for (int t = gt; t < numel; t += gs) {
      T acc = (T)0;
      if (n > 0) {
        const int r = t / n, cc = t - r * n;
        for (int e = 0; e < deg; ++e) {
          const T* ve = vl + (size_t)e * PQ;
          const T* de = d + e * a.W;
          const T u = ph ? ve[poff + r] * de[qoff + cc] : de[poff + r] * ve[a.P + qoff + cc];
          acc += coef[e] * u;
        }
      } else {
        for (int e = 0; e < deg; ++e) acc += coef[e] * d[e * a.W + base + poff + t];
      }
      th[off + t] -= a.gamma * acc;
    }
  }
}

// h = x - alpha_k g into theta, and the deg messages of phase (k + 1) & 1 into the other parity.  One warp per unit: a
// row of a matrix (phase 0: the products h q_e are row dot products), a column (phase 1: h^T p_e, column dot products) or
// kPgVecChunk elements of a 1-D tensor (copied).  The warp steps the unit's elements, then sums each product in the
// lanes' element order and xor butterflies, so a message does not depend on the grid.  Each lane reads back only the
// elements it stepped.
template <typename T>
__global__ void __launch_bounds__(THREADS) pg_step_kernel(const PgArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  const T alpha = c.alpha[ri.k];
  const int ph = ri.par ^ 1;
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * (THREADS / 32);
  T* th = c.theta + (size_t)l * c.n_pad;
  const T* gp = c.grad_part + (size_t)l * c.S * c.n_pad;
  const int PQ = a.P + a.Q;
  const T* vl = a.vec + (size_t)l * c.dmax * PQ;
  const int base = ph ? a.Q : a.P;
  for (int g = blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5);; g += nw) {
    int s = 0, u = g, nu = 0;
    for (; s < a.nseg; ++s) {
      const int* sd = a.seg + 5 * s;
      nu = sd[2] > 0 ? (ph ? sd[2] : sd[1]) : (sd[1] + kPgVecChunk - 1) / kPgVecChunk;
      if (u < nu) break;
      u -= nu;
    }
    if (s == a.nseg) break;
    const int* sd = a.seg + 5 * s;
    const int off = sd[0], m = sd[1], n = sd[2], poff = sd[3], qoff = sd[4];
    int i0, stride, len, vo = 0, mo;
    if (n == 0) {
      i0 = off + u * kPgVecChunk; stride = 1; len = min(kPgVecChunk, m - u * kPgVecChunk);
      mo = base + poff + u * kPgVecChunk;
    } else if (ph == 0) {
      i0 = off + u * n; stride = 1; len = n; vo = a.P + qoff; mo = poff + u;
    } else {
      i0 = off + u; stride = n; len = m; vo = poff; mo = qoff + u;
    }
    for (int j = lane; j < len; j += 32) {
      const size_t i = (size_t)i0 + (size_t)j * stride;
      T gr = gp[i];
      for (int q = 1; q < c.S; ++q) gr += gp[(size_t)q * c.n_pad + i];
      th[i] -= alpha * gr;
    }
    for (int e = 0; e < deg; ++e) {
      T* out = pg_row(a, ri.par ^ 1, e, l) + mo;
      if (n == 0) {
        for (int j = lane; j < len; j += 32) out[j] = th[i0 + j];
        continue;
      }
      const T* ve = vl + (size_t)e * PQ + vo;
      T acc = (T)0;
      for (int j = lane; j < len; j += 32) acc += th[(size_t)i0 + (size_t)j * stride] * ve[j];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) *out = acc;
    }
  }
  end_step(c, l, ri.k, true);
}

// ----------------------------------------------------------- ClippedGossip ----
// Round k (layout and rules in consensus.h): cg_dist, cg_mix, fwd/bwd, cg_step; with `clip: none` dsgd_mix replaces
// the first two.  A clipped edge needs its distance over the whole row before any element is mixed, and the row is
// spread over the CTAs of the node, so the distances take a launch of their own: cg_dist writes one fp64 partial sum
// per fixed chunk of the row, and cg_mix, after the programmatic-dependency wait, adds them in chunk order.
template <typename T>
__global__ void __launch_bounds__(THREADS) cg_dist_kernel(const ClipArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const size_t row = (size_t)l * c.n_pad;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nchunk = cg_chunks(c);
  __shared__ double red[THREADS / 32][4];
  // four neighbors per pass, one partial per chunk of THREADS * N elements with a fixed-order block reduction: the
  // partials, and so the distances, do not depend on the grid (the number of local nodes, the GPU's SM count)
  for (int e0 = 0; e0 < deg; e0 += 4) {
    for (int ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
      const int i = (ch * THREADS + threadIdx.x) * N;
      double s[4] = {0.0, 0.0, 0.0, 0.0};
      if (i < c.n_pad) {
        const Pack<T> th = ldv(c.theta + row + i);
        Pack<T> q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < deg) q[j] = ldv(nbr_row(c, ri.gid, l, e0 + j, ri.par, 0) + i);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < deg) {
#pragma unroll
            for (int u = 0; u < N; ++u) {
              const double d = (double)q[j].v[u] - (double)th.v[u];
              s[j] += d * d;
            }
          }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
        if (lane == 0) red[warp][j] = s[j];
      }
      __syncthreads();
      if ((int)threadIdx.x < 4 && e0 + (int)threadIdx.x < deg) {
        double t = red[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < THREADS / 32; ++w) t += red[w][threadIdx.x];
        a.dist_part[((size_t)l * c.dmax + e0 + threadIdx.x) * a.pstride + ch] = t;
      }
      __syncthreads();
    }
  }
}

// Every CTA of node l sums the distance partials in chunk order (so all of them agree on the distances), thread 0 picks
// the radius: it walks the neighbors from the farthest (ties: the smaller index first) while their Metropolis weights
// sum to at most delta (up to kClipSlack), and tau is the distance of the first neighbor that does not fit (0 when all
// fit).  Then the self-centred mix theta_i + sum_j W_ij min(1, tau / d_ij) (theta_j - theta_i) of the CTA's slice.
template <typename T>
__global__ void __launch_bounds__(THREADS) cg_mix_kernel(const ClipArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  __shared__ double dist[kClipMaxDeg];
  __shared__ T coef[kClipMaxDeg];
  __shared__ bool clipped[kClipMaxDeg];
  for (int e = threadIdx.x; e < deg; e += THREADS) {
    const double* p = a.dist_part + ((size_t)l * c.dmax + e) * a.pstride;
    double s = 0.0;
    const int nchunk = cg_chunks(c);
    for (int b = 0; b < nchunk; ++b) s += p[b];
    dist[e] = sqrt(s);
    clipped[e] = false;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double cum = 0.0, tau = 0.0;
    for (int t = 0; t < deg; ++t) {
      int b = -1;
      for (int e = 0; e < deg; ++e)
        if (!clipped[e] && (b < 0 || dist[e] > dist[b])) b = e;
      if (cum + (double)w[b] > a.delta + kClipSlack) { tau = dist[b]; break; }
      cum += (double)w[b];
      clipped[b] = true;
    }
    for (int e = 0; e < deg; ++e) coef[e] = dist[e] > tau ? (T)((double)w[e] * (tau / dist[e])) : w[e];
  }
  __syncthreads();
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> th0 = ldv(c.theta + row + i);
    Pack<T> th = th0;
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i); },
                     [&](int e, const Pack<T>& q) {
                       const T ce = coef[e];
#pragma unroll
                       for (int u = 0; u < N; ++u) th.v[u] += ce * (q.v[u] - th0.v[u]);
                     });
    stv(c.theta + row + i, th);
  }
}

// ALIE row of a Byzantine node at element i: mu - z sigma, the element-wise mean and population standard deviation
// (fp64) of its honest neighbors' rows of round k; its own theta when it has no honest neighbor.  These are the rows
// cg_mix read this round: the round-start wait that covered those reads still holds, because no neighbor overwrites
// them before this node has published round k + 1 (DESIGN §2.8).
template <typename T>
NNDT_DEVINL Pack<T> alie_row(const ClipArgs<T>& a, const RoundInfo<T>& ri, int l, int i, const Pack<T>& th) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int deg = c.deg[ri.gid * c.L + l];
  const int* byz = a.nbr_byz + (size_t)(ri.gid * c.L + l) * c.dmax;
  double mu[N], var[N];
#pragma unroll
  for (int u = 0; u < N; ++u) mu[u] = var[u] = 0.0;
  int h = 0;
  for (int e = 0; e < deg; ++e)
    if (!byz[e]) {
      const Pack<T> q = ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i);
#pragma unroll
      for (int u = 0; u < N; ++u) mu[u] += (double)q.v[u];
      ++h;
    }
  if (h == 0) return th;
#pragma unroll
  for (int u = 0; u < N; ++u) mu[u] /= (double)h;
  for (int e = 0; e < deg; ++e)
    if (!byz[e]) {
      const Pack<T> q = ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i);
#pragma unroll
      for (int u = 0; u < N; ++u) {
        const double d = (double)q.v[u] - mu[u];
        var[u] += d * d;
      }
    }
  Pack<T> r;
#pragma unroll
  for (int u = 0; u < N; ++u) r.v[u] = (T)(mu[u] - a.z * sqrt(var[u] / (double)h));
  return r;
}

// dsgd_step's arithmetic, written out identically; with ATK a node's attack code picks the row it publishes: theta
// (honest), -scale theta (sign flip) or the ALIE row.  ATK is false on a rank that hosts no attacker.
template <typename T, int U, bool ATK>
__global__ void __launch_bounds__(THREADS) cg_step_kernel(const ClipArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  const int atk = ATK ? a.attack[l] : (int)kHonest;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> th = ldv(c.theta + row + i);
    const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] -= alpha * g.v[u];
    stv(c.theta + row + i, th);
    if (atk == kHonest) {
      stv(pub_row(c, ri.par ^ 1, 0, l) + i, th);
    } else if (atk == kSignFlip) {
      const T s = (T)a.scale;
      Pack<T> p;
#pragma unroll
      for (int u = 0; u < N; ++u) p.v[u] = -(s * th.v[u]);
      stv(pub_row(c, ri.par ^ 1, 0, l) + i, p);
    }
  }
  // the ALIE rows in a loop of their own, over the thread's own stores of theta: inside the step loop the fp64
  // square root's slow-path call spilled the gradient loads
  if (atk == kAlie)
    for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N)
      stv(pub_row(c, ri.par ^ 1, 0, l) + i, alie_row(a, ri, l, i, ldv(c.theta + row + i)));
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------------ BRIDGE ----
// Round k (layout and rules in consensus.h): bridge_mix, fwd/bwd, cg_step.  Each thread screens the elements of its
// 16-byte vector one component at a time: the D neighbor values (+inf in the slots past deg) go through Batcher's
// odd-even merge network (5, 19 or 63 compare-exchanges for D = 4, 8, 16), then fully unrolled, predicated loops over
// static positions sum the kept ones or pick the median, so nothing is indexed dynamically and no value leaves the
// registers.  The median places the own value by its rank among the sorted neighbors instead of sorting D + 1 values.
// Sorted values do not depend on the neighbor table order, so neither does the result (up to the sign of a zero).
template <typename T>
NNDT_DEVINL void cmp_swap(T& x, T& y) {
  const T lo = y < x ? y : x, hi = y < x ? x : y;
  x = lo;
  y = hi;
}

// Batcher's network written as template recursion, so every index is a compile-time constant (the nested loop form
// was not fully unrolled and put the values on the stack)
template <int I, int END, int STEP, int R, int D, typename T>
NNDT_DEVINL void oe_merge_cmp(T (&v)[D]) {
  if constexpr (I < END) {
    cmp_swap(v[I], v[I + R]);
    oe_merge_cmp<I + STEP, END, STEP, R>(v);
  }
}

// merge the two sorted halves of v[LO, LO + N) compared at distance R
template <int LO, int N, int R, int D, typename T>
NNDT_DEVINL void oe_merge(T (&v)[D]) {
  if constexpr (2 * R < N) {
    oe_merge<LO, N, 2 * R>(v);
    oe_merge<LO + R, N, 2 * R>(v);
    oe_merge_cmp<LO + R, LO + N - R, 2 * R, R>(v);
  } else {
    cmp_swap(v[LO], v[LO + R]);
  }
}

template <int LO, int N, int D, typename T>
NNDT_DEVINL void oe_sort(T (&v)[D]) {
  if constexpr (N > 1) {
    oe_sort<LO, N / 2>(v);
    oe_sort<LO + N / 2, N / 2>(v);
    oe_merge<LO, N, 1>(v);
  }
}

template <int D, typename T>
NNDT_DEVINL void odd_even_merge_sort(T (&v)[D]) {
  static_assert((D & (D - 1)) == 0, "the network sorts a power of two");
  oe_sort<0, D>(v);
}

// merged position q of the own value x (rank r among the sorted neighbors s) and s
template <int D, typename T>
NNDT_DEVINL T merged_at(const T (&s)[D], T x, int r, int q) {
  T out = x;
#pragma unroll
  for (int p = 0; p < D; ++p) {
    if (p < r && p == q) out = s[p];
    if (p >= r && p + 1 == q) out = s[p];
  }
  return out;
}

// -Xptxas -v, no spills and no stack: 58 / 88 / 122 registers for fp64 with 4 / 8 / 16 slots, 66 / 86 / 136 for fp32.
// Without the minimum of one CTA per SM ptxas held the fp32 16-slot variant to 128 registers and spilled.
template <typename T, int D>
__global__ void __launch_bounds__(THREADS, 1) bridge_mix_kernel(const ScreenArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const int lo = a.b, hi = deg - a.b;                        // trimmed mean: kept sorted positions [lo, hi)
  const double kept = 1.0 + (double)max(0, hi - lo);
  const int ql = deg / 2, qh = (deg + 1) / 2;                 // median: middle merged positions of deg + 1 values
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> th = ldv(c.theta + row + i);
    Pack<T> q[D];
#pragma unroll
    for (int e = 0; e < D; ++e) {
      if (e < deg) {
        q[e] = ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i);
      } else {
#pragma unroll
        for (int u = 0; u < N; ++u) q[e].v[u] = (T)INFINITY;
      }
    }
    Pack<T> y;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      T s[D];
#pragma unroll
      for (int e = 0; e < D; ++e) s[e] = q[e].v[u];
      odd_even_merge_sort<D>(s);
      const T x = th.v[u];
      if (a.median) {
        int r = 0;
#pragma unroll
        for (int p = 0; p < D; ++p) r += s[p] < x ? 1 : 0;
        const T vl = merged_at<D>(s, x, r, ql), vh = merged_at<D>(s, x, r, qh);
        y.v[u] = ql == qh ? vl : (T)(0.5 * ((double)vl + (double)vh));
      } else {
        double acc = (double)x;
#pragma unroll
        for (int p = 0; p < D; ++p)
          if (p >= lo && p < hi) acc += (double)s[p];
        y.v[u] = (T)div_rn(acc, kept);
      }
    }
    stv(c.theta + row + i, y);
  }
}

// -------------------------------------------------------------------- SGP ----
// Round k: sgp_mix pulls the in-neighbors' rows (x, w) of round k, x_i <- sum_j A_ij x_j, w_i <- sum_j A_ij w_j,
// theta_i <- x_i / w_i; sgp_step takes x_i -= alpha_k g_i(theta_i), theta_i <- x_i / w_i and publishes (x_i, w_i).
template <typename T>
__global__ void __launch_bounds__(THREADS) sgp_mix_kernel(const SgpArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  // the new push-sum weight, from the node's own published row (a.w[l] is stored below): every CTA of the node sums
  // in the same order, so all of them divide by the same bits
  double wn = (double)ws * row_weight(sgp_row(a, ri.par, l), c.n_pad);
  for_neighbors<4>(deg, [&](int e) { return row_weight(nbr_row(c, ri.gid, l, e, ri.par, 0), c.n_pad); },
                   [&](int e, double q) { wn += (double)w[e] * q; });
  if (blockIdx.x == 0 && threadIdx.x == 0) a.w[l] = wn;
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> x = ldv(a.x + row + i);
#pragma unroll
    for (int u = 0; u < N; ++u) x.v[u] *= ws;
    for_neighbors<4>(deg, [&](int e) { return ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i); },
                     [&](int e, const Pack<T>& q) {
#pragma unroll
                       for (int u = 0; u < N; ++u) x.v[u] += w[e] * q.v[u];
                     });
    Pack<T> th;
#pragma unroll
    for (int u = 0; u < N; ++u) th.v[u] = sgp_debias(x.v[u], wn);
    stv(a.x + row + i, x);
    stv(c.theta + row + i, th);
  }
}

template <typename T, int U>
__global__ void __launch_bounds__(THREADS) sgp_step_kernel(const SgpArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const T alpha = c.alpha[ri.k];
  const size_t row = (size_t)l * c.n_pad;
  T* out = sgp_row(a, ri.par ^ 1, l);
  // w and x (written by the mix two launches back) are read before the programmatic-dependency wait; only the
  // gradient partials of the forward/backward kernel after it
  const double wn = a.w[l];
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    Pack<T> x = ldv(a.x + row + i);
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
    Pack<T> th;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      x.v[u] -= alpha * g.v[u];
      th.v[u] = sgp_debias(x.v[u], wn);
    }
    stv(a.x + row + i, x);
    stv(c.theta + row + i, th);
    stv(out + i, x);
  }
  release_dependents_once(waited);
  if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<double*>(out + c.n_pad) = wn;
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------- Push-DIGing ----
// Round k: pdg_mix pulls each in-neighbor's u row, y row and w tail of round k once,
//   u_i <- sum_j A_ij (u_j - alpha y_j),  ysum_i <- sum_j A_ij y_j,  w_i <- sum_j A_ij w_j,  theta_i <- u_i / w_i;
// pdg_track forms y_i <- ysum_i + (g_i - g_old_i) from the local rows and publishes (u_i, w_i) and y_i.  Every neighbor
// read of the round happens in the mix, after begin_round, as in SGP.
template <typename T>
struct UYPack { Pack<T> u, y; };

template <typename T>
__global__ void __launch_bounds__(THREADS) pdg_mix_kernel(const PushDigArgs<T> a) {
  pdl_wait();
  pdl_launch_dependents();
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const int deg = c.deg[ri.gid * c.L + l];
  begin_round(c, ri.gid, l, ri.k);
  const T alpha = c.alpha[ri.k];
  const T ws = c.self_w[ri.gid * c.L + l];
  const T* w = c.nbr_w + (size_t)(ri.gid * c.L + l) * c.dmax;
  const T* ys = pdg_row(a, ri.par, 1, l);
  // the new push-sum weight, summed in one order by every CTA of the node (as in sgp_mix): all divide by the same bits
  double wn = (double)ws * row_weight(pdg_row(a, ri.par, 0, l), c.n_pad);
  for_neighbors<4>(deg, [&](int e) { return row_weight(nbr_row(c, ri.gid, l, e, ri.par, 0), c.n_pad); },
                   [&](int e, double q) { wn += (double)w[e] * q; });
  if (blockIdx.x == 0 && threadIdx.x == 0) a.w[l] = wn;
  const size_t row = (size_t)l * c.n_pad;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> y = ldv(ys + i);
    Pack<T> u = ldv(a.u + row + i), s;
#pragma unroll
    for (int v = 0; v < N; ++v) {
      u.v[v] = ws * (u.v[v] - alpha * y.v[v]);
      s.v[v] = ws * y.v[v];
    }
    for_neighbors<2>(deg,
                     [&](int e) {
                       return UYPack<T>{ldv(nbr_row(c, ri.gid, l, e, ri.par, 0) + i),
                                        ldv(nbr_row(c, ri.gid, l, e, ri.par, 1) + i)};
                     },
                     [&](int e, const UYPack<T>& q) {
                       const T we = w[e];
#pragma unroll
                       for (int v = 0; v < N; ++v) {
                         u.v[v] += we * (q.u.v[v] - alpha * q.y.v[v]);
                         s.v[v] += we * q.y.v[v];
                       }
                     });
    Pack<T> th;
#pragma unroll
    for (int v = 0; v < N; ++v) th.v[v] = sgp_debias(u.v[v], wn);
    stv(a.u + row + i, u);
    stv(c.theta + row + i, th);
    stv(a.ysum + row + i, s);
  }
}

template <typename T, int U>
__global__ void __launch_bounds__(THREADS) pdg_track_kernel(const PushDigArgs<T> a) {
  const Common<T>& c = a.c;
  constexpr int N = Vec<T>::N;
  const int l = node_of_block(c);
  const RoundInfo<T> ri = round_info(c);
  const size_t row = (size_t)l * c.n_pad;
  T* ou = pdg_row(a, ri.par ^ 1, 0, l);
  T* oy = pdg_row(a, ri.par ^ 1, 1, l);
  // u, ysum and w (written by the mix two launches back) and g_old (the previous round) are read before the
  // programmatic-dependency wait; only the gradient partials of the forward/backward kernel after it
  const double wn = a.w[l];
  bool waited = false;
  for (int i = (blockIdx.x * THREADS + threadIdx.x) * N; i < c.n_pad; i += gridDim.x * THREADS * N) {
    const Pack<T> u = ldv(a.u + row + i);
    Pack<T> y = ldv(a.ysum + row + i);
    const Pack<T> go = ldv(a.g_old + row + i);
    release_dependents_once(waited);
    const Pack<T> g = sum_partials<U>(c, l, i);
#pragma unroll
    for (int v = 0; v < N; ++v) y.v[v] += g.v[v] - go.v[v];
    stv(a.g_old + row + i, g);
    stv(oy + i, y);
    stv(ou + i, u);
  }
  release_dependents_once(waited);
  if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<double*>(ou + c.n_pad) = wn;
  end_step(c, l, ri.k, true);
}

// ------------------------------------------------------------ consensus metric ----
NNDT_DEVINL double block_sum(double v) {
  __shared__ double red[THREADS / 32];
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < THREADS / 32; ++w) t += red[w];
  return t;
}
template <typename T>
__global__ void __launch_bounds__(THREADS) inv_norm_kernel(const int64_t* rows, int n_pad, double* inv_norm) {
  const T* r = reinterpret_cast<const T*>(rows[blockIdx.x]);
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_pad; i += THREADS) { const double v = (double)r[i]; acc += v * v; }
  acc = block_sum(acc);
  if (threadIdx.x == 0) inv_norm[blockIdx.x] = 1.0 / fmax(sqrt(acc), 1e-12);   // F.normalize eps
}
// block (j, l): j < N -> pair distance to node j;  j == N -> distance to the mean of the normalised rows
template <typename T>
__global__ void __launch_bounds__(THREADS) consensus_metric_kernel(const int64_t* rows, int N, int n_pad, int local0,
                                                                   const double* inv_norm, double* out_pair, double* out_mean) {
  const int j = blockIdx.x, l = blockIdx.y, gi = local0 + l;
  const T* ri = reinterpret_cast<const T*>(rows[gi]);
  const double ni = inv_norm[gi];
  double acc = 0.0;
  if (j < N) {
    const T* rj = reinterpret_cast<const T*>(rows[j]);
    const double nj = inv_norm[j];
    for (int e = threadIdx.x; e < n_pad; e += THREADS) {
      const double d = (double)ri[e] * ni - (double)rj[e] * nj;
      acc += d * d;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) out_pair[(size_t)l * N + j] = sqrt(acc);
  } else {
    for (int e = threadIdx.x; e < n_pad; e += THREADS) {
      double mu = 0.0;
      for (int q = 0; q < N; ++q) mu += (double)reinterpret_cast<const T*>(rows[q])[e] * inv_norm[q];
      const double d = (double)ri[e] * ni - mu / (double)N;
      acc += d * d;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) out_mean[l] = sqrt(acc);
  }
}
template <typename T>
cudaError_t launch_consensus_metric(const int64_t* rows, int N, int n_pad, int local0, int L, double* inv_norm,
                                    double* out_pair, double* out_mean, cudaStream_t st) {
  inv_norm_kernel<T><<<N, THREADS, 0, st>>>(rows, n_pad, inv_norm);
  consensus_metric_kernel<T><<<dim3(N + 1, L), THREADS, 0, st>>>(rows, N, n_pad, local0, inv_norm, out_pair, out_mean);
  return cudaGetLastError();
}

// ------------------------------------------------------------ rank barrier ----
__global__ void rank_barrier_kernel(int* slots, const int64_t* peer_slot, int world, int rank, int epoch,
                                    const volatile int* gate, int* err) {
  if (gate != nullptr && threadIdx.x == 0) {
    const long long t0 = clock64();
    while (*gate == 0) {
      if (clock64() - t0 > kSpinLimit) { if (err) *err = 1; break; }
    }
  }
  __syncthreads();
  const int r = threadIdx.x;
  if (r < world && r != rank) {
    __threadfence_system();
    st_release_sys(reinterpret_cast<int*>(peer_slot[r]), epoch);
    const long long t0 = clock64();
    while (ld_acquire_sys(slots + r) < epoch) {
      if (clock64() - t0 > kSpinLimit) { if (err) *err = 1; break; }
    }
  }
}
cudaError_t launch_rank_barrier(int* slots, const int64_t* peer_slot, int world, int rank, int epoch,
                                const volatile int* gate, int* err, cudaStream_t st) {
  rank_barrier_kernel<<<1, 64, 0, st>>>(slots, peer_slot, world, rank, epoch, gate, err);
  return cudaGetLastError();
}
__global__ void spin_kernel(long long cycles) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
}
cudaError_t launch_spin(long long cycles, cudaStream_t st) {
  spin_kernel<<<1, 1, 0, st>>>(cycles);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- launchers ----
// One wave: the grid of an update kernel is capped at the number of CTAs that can be resident at once (the kernels
// loop over the row with a grid stride).  A second wave costs a full CTA start-up + the dependent header loads
// (round counter -> schedules -> topology -> data, ~4 L2 round trips), more than a second loop iteration does.
template <typename K>
static int resident_ctas(K kernel) {
  static std::mutex mu;
  static std::unordered_map<const void*, int> cache;       // per kernel instantiation (one device type per process)
  std::lock_guard<std::mutex> lock(mu);
  const void* key = reinterpret_cast<const void*>(kernel);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  int dev = 0, sms = 0, occ = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, THREADS, 0) != cudaSuccess || occ < 1) occ = 1;
  return cache[key] = sms * occ;
}
template <typename T, typename K>
static dim3 grid_for(const Common<T>& c, K kernel) {
  const int per_block = THREADS * Vec<T>::N;
  int gx = (c.n_pad + per_block - 1) / per_block;
  const int slots = resident_ctas(kernel);
  if (gx * c.L > slots) {
    const int iters = (gx * c.L + slots - 1) / slots;       // loop iterations per thread that make it fit
    gx = (gx + iters - 1) / iters;
  }
  return dim3(gx > 0 ? gx : 1, c.L);
}

template <typename T> cudaError_t launch_local_sum(const Common<T>& c, cudaStream_t st) {
  const int per_block = THREADS * Vec<T>::N;
  return launch_pdl(local_sum_kernel<T>, dim3((c.n_pad + per_block - 1) / per_block), dim3(THREADS), 0, st, c);
}
template <typename T, typename K, typename A>
static cudaError_t launch_one_wave(K kernel, const Common<T>& c, const A& a, cudaStream_t st) {
  return launch_pdl(kernel, grid_for(c, kernel), dim3(THREADS), 0, st, a);
}
// kernels that sum gradient partials: the shallow variant (4 loads in flight) when the producer writes <= 4 partial
// rows per node, the deep one otherwise
template <typename T, typename K, typename A>
static cudaError_t launch_by_s(K shallow, K deep, const Common<T>& c, const A& a, cudaStream_t st) {
  return launch_one_wave(c.S <= 4 ? shallow : deep, c, a, st);
}
template <typename T> cudaError_t launch_dinno_update(const DinnoArgs<T>& a, cudaStream_t st) {
  return launch_by_s(dinno_update_kernel<T, 4>, dinno_update_kernel<T, 16>, a.c, a, st);
}
template <typename T> cudaError_t launch_local_step(const LocalArgs<T>& a, cudaStream_t st) {
  return launch_by_s(local_step_kernel<T, 4>, local_step_kernel<T, 16>, a.c, a, st);
}
template <typename T> cudaError_t launch_dsgd_mix(const Common<T>& c, cudaStream_t st) {
  return launch_one_wave(dsgd_mix_kernel<T>, c, c, st);
}
template <typename T> cudaError_t launch_dsgd_step(const Common<T>& c, cudaStream_t st) {
  return launch_by_s(dsgd_step_kernel<T, 4>, dsgd_step_kernel<T, 16>, c, c, st);
}
template <typename T> cudaError_t launch_dsgt_init(const DsgtArgs<T>& a, cudaStream_t st) {
  return launch_by_s(dsgt_init_kernel<T, 4>, dsgt_init_kernel<T, 16>, a.c, a, st);
}
template <typename T> cudaError_t launch_dsgt_mix(const DsgtArgs<T>& a, cudaStream_t st) {
  // the own-tracker step is a template parameter: as a runtime branch it raised the register count past the
  // 64 per thread that keep 4 CTAs resident per SM
  return launch_one_wave(a.own_tracker ? dsgt_mix_kernel<T, true> : dsgt_mix_kernel<T, false>, a.c, a, st);
}
template <typename T> cudaError_t launch_dsgt_track(const DsgtArgs<T>& a, cudaStream_t st) {
  return launch_by_s(dsgt_track_kernel<T, 4>, dsgt_track_kernel<T, 16>, a.c, a, st);
}
template <typename T> cudaError_t launch_ed_mix(const EdArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(a.c.sum_mode ? ed_sum_mix_kernel<T> : dsgd_mix_kernel<T>, a.c, a.c, st);
}
template <typename T> cudaError_t launch_ed_step(const EdArgs<T>& a, cudaStream_t st) {
  return launch_by_s(ed_step_kernel<T, 4>, ed_step_kernel<T, 16>, a.c, a, st);
}
// the momentum mode and Nesterov are template parameters, not runtime branches (see dsgt_mix above).  Beyond 4 gradient
// partials the step keeps 8 loads in flight, as sgp_step: 16 spilled in fp32
template <typename T, bool QG, bool NEST> static cudaError_t launch_dsgdm(const MomentumArgs<T>& a, cudaStream_t st) {
  return launch_by_s(dsgdm_step_kernel<T, 4, QG, NEST>, dsgdm_step_kernel<T, 8, QG, NEST>, a.c, a, st);
}
template <typename T> cudaError_t launch_dsgdm_step(const MomentumArgs<T>& a, cudaStream_t st) {
  if (a.x_prev != nullptr) return a.nesterov ? launch_dsgdm<T, true, true>(a, st) : launch_dsgdm<T, true, false>(a, st);
  return a.nesterov ? launch_dsgdm<T, false, true>(a, st) : launch_dsgdm<T, false, false>(a, st);
}
// the compressor is a template parameter, not a runtime branch (see dsgt_mix above).  With more than 4 gradient
// partials the step keeps 8 loads in flight (the summation order is the same for any depth); 16, as the other step
// kernels use, took 164 registers (fp64) or spilled (fp32) next to the encoder
template <typename T, int Q> static cudaError_t launch_choco_q(const ChocoArgs<T>& a, bool step, cudaStream_t st) {
  return step ? launch_by_s(choco_step_kernel<T, 4, Q>, choco_step_kernel<T, 8, Q>, a.c, a, st)
              : launch_one_wave(choco_mix_kernel<T, Q>, a.c, a, st);
}
// top-k step: one cluster of kTopkCluster CTAs per node, grid (CS, L), with `chans` slices of v in dynamic shared memory
template <typename T, typename K, typename A>
static cudaError_t launch_topk_step(K kernel, const Common<T>& c, int chans, int k, long long stride, const A& a,
                                    cudaStream_t st) {
  const int sl = topk_slice(c.n_pad);
  const size_t smem = (size_t)chans * sl * sizeof(T) + sl / 8;      // the slices of v, then the slice's live words
  if (smem > (size_t)kTopkRowSmem || k < 1 || stride < (long long)k * (long long)(sizeof(T) + 4)) return cudaErrorInvalidValue;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTopkRowSmem);
  if (e != cudaSuccess) return e;
  return launch_pdl_cluster(kernel, dim3(kTopkCluster, c.L), dim3(THREADS), smem, kTopkCluster, st, a);
}
template <typename T> static cudaError_t launch_choco(const ChocoArgs<T>& a, bool step, cudaStream_t st) {
  switch (a.code) {
    case kCodeNone: return launch_choco_q<T, kCodeNone>(a, step, st);
    case kCodeInt8: return launch_choco_q<T, kCodeInt8>(a, step, st);
    case kCodeSign: return launch_choco_q<T, kCodeSign>(a, step, st);
    case kCodeTopk:
      if (!step) return launch_one_wave(choco_topk_mix_kernel<T>, a.c, a, st);
      return launch_topk_step(a.c.S <= 4 ? choco_topk_step_kernel<T, 4> : choco_topk_step_kernel<T, 8>, a.c, 1, a.topk_k,
                              a.code_stride, a, st);
  }
  return cudaErrorInvalidValue;
}
template <typename T> cudaError_t launch_choco_mix(const ChocoArgs<T>& a, cudaStream_t st) { return launch_choco(a, false, st); }
template <typename T> cudaError_t launch_choco_step(const ChocoArgs<T>& a, cudaStream_t st) { return launch_choco(a, true, st); }
// as CHOCO: the compressor is a template parameter, and beyond 4 gradient partials the step keeps 8 loads in flight
template <typename T, int Q> static cudaError_t launch_beer_q(const BeerArgs<T>& a, bool step, cudaStream_t st) {
  return step ? launch_by_s(beer_step_kernel<T, 4, Q>, beer_step_kernel<T, 8, Q>, a.c, a, st)
              : launch_one_wave(beer_mix_kernel<T, Q>, a.c, a, st);
}
template <typename T> static cudaError_t launch_beer(const BeerArgs<T>& a, bool step, cudaStream_t st) {
  switch (a.code) {
    case kCodeNone: return launch_beer_q<T, kCodeNone>(a, step, st);
    case kCodeInt8: return launch_beer_q<T, kCodeInt8>(a, step, st);
    case kCodeSign: return launch_beer_q<T, kCodeSign>(a, step, st);
    case kCodeTopk:
      if (!step) return launch_one_wave(beer_topk_mix_kernel<T>, a.c, a, st);
      return launch_topk_step(a.c.S <= 4 ? beer_topk_step_kernel<T, 4> : beer_topk_step_kernel<T, 8>, a.c, 2, a.topk_k,
                              a.code_stride, a, st);
  }
  return cudaErrorInvalidValue;
}
template <typename T> cudaError_t launch_beer_mix(const BeerArgs<T>& a, cudaStream_t st) { return launch_beer(a, false, st); }
template <typename T> cudaError_t launch_beer_step(const BeerArgs<T>& a, cudaStream_t st) { return launch_beer(a, true, st); }

template <typename T> cudaError_t launch_kgt_mix(const KgtArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(kgt_mix_kernel<T>, a.c, a, st);
}
// the correction is a template parameter (see dsgt_mix above); beyond 4 gradient partials the step keeps 8 loads in
// flight, as sgp_step
template <typename T, bool CORR> static cudaError_t launch_kgt(const KgtArgs<T>& a, cudaStream_t st) {
  return launch_by_s(kgt_step_kernel<T, 4, CORR>, kgt_step_kernel<T, 8, CORR>, a.c, a, st);
}
template <typename T> cudaError_t launch_kgt_step(const KgtArgs<T>& a, cudaStream_t st) {
  return a.correction ? launch_kgt<T, true>(a, st) : launch_kgt<T, false>(a, st);
}

template <typename T> cudaError_t launch_ag_gossip(const DetagArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(a.step == a.K - 1 ? ag_gossip_kernel<T, true> : ag_gossip_kernel<T, false>, a.c, a, st);
}
template <typename T> cudaError_t launch_detag_track(const DetagArgs<T>& a, cudaStream_t st) {
  return launch_by_s(detag_track_kernel<T, 4>, detag_track_kernel<T, 8>, a.c, a, st);
}
template <typename T> cudaError_t launch_hsgd_track(const HsgdArgs<T>& a, cudaStream_t st) {
  // 8-deep as detag_track (S > 8 runs the tail loop): with two partial sets the 16-deep fp32 variant spills
  return launch_by_s(hsgd_track_kernel<T, 4>, hsgd_track_kernel<T, 8>, a.c, a, st);
}
template <typename T> cudaError_t launch_xg_pull(const XgArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(xg_pull_kernel<T>, a.c, a, st);
}
template <typename T> cudaError_t launch_xg_publish(const XgArgs<T>& a, cudaStream_t st) {
  return launch_by_s(xg_publish_kernel<T, 4>, xg_publish_kernel<T, 8>, a.c, a, st);
}
template <typename T> cudaError_t launch_xg_step(const XgArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(xg_step_kernel<T>, a.c, a, st);
}

// pga_sum covers the row once, one CTA per THREADS vectors, as local_sum; pga_mix is one wave, as dsgd_mix
template <typename T> cudaError_t launch_pga_sum(const PgaArgs<T>& a, cudaStream_t st) {
  if (a.period < 1 || a.c.sum_local == nullptr || a.c.C != 1 || a.c.sum_mode) return cudaErrorInvalidValue;
  const int per_block = THREADS * Vec<T>::N;
  return launch_pdl(pga_sum_kernel<T>, dim3((a.c.n_pad + per_block - 1) / per_block), dim3(THREADS), 0, st, a);
}
template <typename T> cudaError_t launch_pga_mix(const PgaArgs<T>& a, cudaStream_t st) {
  if (a.period < 1 || a.c.sum_local == nullptr || a.c.C != 1 || a.c.sum_mode || a.c.n_total < 1)
    return cudaErrorInvalidValue;
  return launch_one_wave(pga_mix_kernel<T>, a.c, a, st);
}
// one wave over the local rows, as dsgd_step
template <typename T> cudaError_t launch_slowmo_outer(const SlowmoArgs<T>& a, cudaStream_t st) {
  if (a.period < 1 || a.anchor == nullptr || a.u == nullptr || a.c.C != 1) return cudaErrorInvalidValue;
  return launch_one_wave(slowmo_outer_kernel<T>, a.c, a, st);
}

// dp_norm and dp_step: one wave each, the 8-deep partial sum beyond 4 partials (as sgp_step)
template <typename T> static bool dp_ready(const DpArgs<T>& a) {
  return a.norm_part != nullptr && a.pstride >= cg_chunks(a.c) && a.nbr_id != nullptr && a.live != nullptr &&
         a.c.C == 1 && !a.c.sum_mode;
}
template <typename T> cudaError_t launch_dp_norm(const DpArgs<T>& a, cudaStream_t st) {
  if (!dp_ready(a)) return cudaErrorInvalidValue;
  return launch_by_s(dp_norm_kernel<T, 4>, dp_norm_kernel<T, 8>, a.c, a, st);
}
template <typename T> cudaError_t launch_dp_step(const DpArgs<T>& a, cudaStream_t st) {
  if (!dp_ready(a)) return cudaErrorInvalidValue;
  return launch_by_s(dp_step_kernel<T, 4>, dp_step_kernel<T, 8>, a.c, a, st);
}

// mq_mix and mq_step: the bit width and the base are template parameters; beyond 4 gradient partials the step keeps 8
// loads in flight (as choco_step)
template <typename T> static bool mq_ready(const MoniquaArgs<T>& a) {
  return (a.bits == 2 || a.bits == 4 || a.bits == 8) && a.live != nullptr && a.margin != nullptr && a.B > 0.0 &&
         a.c.n_pad % 128 == 0 && a.code_stride == (long long)a.c.n_pad * a.bits / 8 && a.c.C == 1 && !a.c.sum_mode;
}
template <typename T, int BITS> static cudaError_t launch_mq_bits(const MoniquaArgs<T>& a, bool step, cudaStream_t st) {
  if (!step) return launch_one_wave(mq_mix_kernel<T, BITS>, a.c, a, st);
  if (a.psi != nullptr) return launch_by_s(mq_step_kernel<T, 4, BITS, true>, mq_step_kernel<T, 8, BITS, true>, a.c, a, st);
  return launch_by_s(mq_step_kernel<T, 4, BITS, false>, mq_step_kernel<T, 8, BITS, false>, a.c, a, st);
}
template <typename T> static cudaError_t launch_mq(const MoniquaArgs<T>& a, bool step, cudaStream_t st) {
  if (!mq_ready(a)) return cudaErrorInvalidValue;
  switch (a.bits) {
    case 2: return launch_mq_bits<T, 2>(a, step, st);
    case 4: return launch_mq_bits<T, 4>(a, step, st);
    default: return launch_mq_bits<T, 8>(a, step, st);
  }
}
template <typename T> cudaError_t launch_mq_mix(const MoniquaArgs<T>& a, cudaStream_t st) { return launch_mq(a, false, st); }
template <typename T> cudaError_t launch_mq_step(const MoniquaArgs<T>& a, cudaStream_t st) { return launch_mq(a, true, st); }

// sparq_mix and sparq_publish: the compressor is a template parameter, one wave each (as choco_mix); sparq_step keeps 8
// gradient loads in flight beyond 4 partials (as kgt_step), and the last step is a variant of its own
template <typename T> static bool sparq_ready(const SparqArgs<T>& a) {
  return a.x_hat != nullptr && a.s != nullptr && a.live != nullptr && a.thr != nullptr && a.norm_part != nullptr &&
         a.triggers != nullptr && a.pstride >= cg_chunks(a.c) && a.H >= 1 && a.code_bytes > 0 && a.code_bytes % 16 == 0 &&
         a.row_stride == a.code_bytes + 16 && a.c.n_pad % 128 == 0 && a.c.dmax <= THREADS && a.c.C == 1 &&
         !a.c.sum_mode && (a.code == kCodeNone || a.code == kCodeInt8 || a.code == kCodeSign);
}
template <typename T, int Q> static cudaError_t launch_sparq_q(const SparqArgs<T>& a, bool publish, cudaStream_t st) {
  return launch_one_wave(publish ? sparq_publish_kernel<T, Q> : sparq_mix_kernel<T, Q>, a.c, a, st);
}
template <typename T> static cudaError_t launch_sparq(const SparqArgs<T>& a, bool publish, cudaStream_t st) {
  if (!sparq_ready(a)) return cudaErrorInvalidValue;
  switch (a.code) {
    case kCodeNone: return launch_sparq_q<T, kCodeNone>(a, publish, st);
    case kCodeInt8: return launch_sparq_q<T, kCodeInt8>(a, publish, st);
    default: return launch_sparq_q<T, kCodeSign>(a, publish, st);
  }
}
template <typename T> cudaError_t launch_sparq_mix(const SparqArgs<T>& a, cudaStream_t st) { return launch_sparq(a, false, st); }
template <typename T> cudaError_t launch_sparq_publish(const SparqArgs<T>& a, cudaStream_t st) { return launch_sparq(a, true, st); }
template <typename T> cudaError_t launch_sparq_step(const SparqArgs<T>& a, cudaStream_t st) {
  if (!sparq_ready(a) || a.step < 0 || a.step >= a.H) return cudaErrorInvalidValue;
  if (a.step == a.H - 1) return launch_by_s(sparq_step_kernel<T, 4, true>, sparq_step_kernel<T, 8, true>, a.c, a, st);
  return launch_by_s(sparq_step_kernel<T, 4, false>, sparq_step_kernel<T, 8, false>, a.c, a, st);
}

template <typename T> cudaError_t launch_dadaptive_mix(const DAdaptiveArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(dadaptive_mix_kernel<T>, a.c, a, st);
}
// the variant and the tracking are template parameters (see dsgt_mix above); beyond 4 gradient partials the step keeps
// 8 loads in flight, as kgt_step
template <typename T, bool ADAGRAD, bool TRACK>
static cudaError_t launch_dadaptive(const DAdaptiveArgs<T>& a, cudaStream_t st) {
  return launch_by_s(dadaptive_step_kernel<T, 4, ADAGRAD, TRACK>, dadaptive_step_kernel<T, 8, ADAGRAD, TRACK>, a.c, a, st);
}
template <typename T> cudaError_t launch_dadaptive_step(const DAdaptiveArgs<T>& a, cudaStream_t st) {
  if (a.adagrad) return a.tracking ? launch_dadaptive<T, true, true>(a, st) : launch_dadaptive<T, true, false>(a, st);
  return a.tracking ? launch_dadaptive<T, false, true>(a, st) : launch_dadaptive<T, false, false>(a, st);
}

template <typename T> cudaError_t launch_relay_mix(const RelayArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(relay_mix_kernel<T>, a.c, a, st);
}
// the received rows stay in registers: 4 of them for paths and binary trees, kRelayMaxDeg up to a star hub.  With at most
// 4 neighbors and more than 4 gradient partials the step keeps 8 loads in flight, as kgt_step; the 16-slot variant keeps
// 4 (the summation order is the same for any depth)
template <typename T> cudaError_t launch_relay_step(const RelayArgs<T>& a, cudaStream_t st) {
  if (a.c.dmax > kRelayMaxDeg) return cudaErrorInvalidValue;
  if (a.c.dmax > 4) return launch_one_wave(relay_step_kernel<T, 4, kRelayMaxDeg>, a.c, a, st);
  return launch_by_s(relay_step_kernel<T, 4, 4>, relay_step_kernel<T, 8, 4>, a.c, a, st);
}

// PowerGossip: pg_mix holds the deg message differences in dynamic shared memory (the opt-in limit is checked by
// ops/engine.py: check_powergossip_capacity); the grid is one wave at that footprint, or `grid_x` CTAs per node
template <typename T, typename K>
static cudaError_t launch_pg(K kernel, const PgArgs<T>& a, size_t smem, cudaStream_t st) {
  const Common<T>& c = a.c;
  if (c.dmax > kPgMaxDeg) return cudaErrorInvalidValue;
  int dev = 0, sms = 0, occ = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  int gx = a.grid_x;
  if (gx <= 0) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, THREADS, smem) != cudaSuccess || occ < 1) occ = 1;
    const int per_block = THREADS * Vec<T>::N, slots = sms * occ;
    gx = (c.n_pad + per_block - 1) / per_block;
    if (gx * c.L > slots) {
      const int iters = (gx * c.L + slots - 1) / slots;
      gx = (gx + iters - 1) / iters;
    }
    gx = gx > 0 ? gx : 1;
  }
  return launch_pdl(kernel, dim3(gx, c.L), dim3(THREADS), smem, st, a);
}
template <typename T> cudaError_t launch_pg_mix(const PgArgs<T>& a, cudaStream_t st) {
  return launch_pg(pg_mix_kernel<T>, a, (size_t)a.c.dmax * a.W * sizeof(T), st);
}
template <typename T> cudaError_t launch_pg_step(const PgArgs<T>& a, cudaStream_t st) {
  return launch_pg(pg_step_kernel<T>, a, 0, st);
}

template <typename T> cudaError_t launch_cg_dist(const ClipArgs<T>& a, cudaStream_t st) {
  if (cg_chunks(a.c) > a.pstride) return cudaErrorInvalidValue;
  return launch_one_wave(cg_dist_kernel<T>, a.c, a, st);
}
template <typename T> cudaError_t launch_cg_mix(const ClipArgs<T>& a, cudaStream_t st) {
  if (cg_chunks(a.c) > a.pstride) return cudaErrorInvalidValue;
  return launch_one_wave(cg_mix_kernel<T>, a.c, a, st);
}
// beyond 4 gradient partials the step keeps 8 loads in flight, as sgp_step: 16 spilled in fp32, as dsgd_step's does
// (the summation order is the same for any depth).  A rank with an attacker keeps 4 in flight at any count: the fp32
// 8-deep attack variant spilled around the fp64 square root's slow-path call.
template <typename T> cudaError_t launch_cg_step(const ClipArgs<T>& a, cudaStream_t st) {
  if (a.attack == nullptr) return launch_by_s(cg_step_kernel<T, 4, false>, cg_step_kernel<T, 8, false>, a.c, a, st);
  return launch_one_wave(cg_step_kernel<T, 4, true>, a.c, a, st);
}

// the fewest neighbor slots that hold the plan's largest degree
template <typename T> cudaError_t launch_bridge_mix(const ScreenArgs<T>& a, cudaStream_t st) {
  if (a.c.dmax > kBridgeMaxDeg) return cudaErrorInvalidValue;
  if (a.c.dmax <= 4) return launch_one_wave(bridge_mix_kernel<T, 4>, a.c, a, st);
  if (a.c.dmax <= 8) return launch_one_wave(bridge_mix_kernel<T, 8>, a.c, a, st);
  return launch_one_wave(bridge_mix_kernel<T, kBridgeMaxDeg>, a.c, a, st);
}

template <typename T> cudaError_t launch_sgp_mix(const SgpArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(sgp_mix_kernel<T>, a.c, a, st);
}
// beyond 4 gradient partials the step keeps 8 loads in flight: 16 spilled in fp32 (the summation order is the same)
template <typename T> cudaError_t launch_sgp_step(const SgpArgs<T>& a, cudaStream_t st) {
  return launch_by_s(sgp_step_kernel<T, 4>, sgp_step_kernel<T, 8>, a.c, a, st);
}

template <typename T> cudaError_t launch_pdg_mix(const PushDigArgs<T>& a, cudaStream_t st) {
  return launch_one_wave(pdg_mix_kernel<T>, a.c, a, st);
}
// beyond 4 gradient partials the track keeps 8 loads in flight, as sgp_step: 16 spilled in fp32
template <typename T> cudaError_t launch_pdg_track(const PushDigArgs<T>& a, cudaStream_t st) {
  return launch_by_s(pdg_track_kernel<T, 4>, pdg_track_kernel<T, 8>, a.c, a, st);
}

#define NNDT_INST(T)                                                                  \
  template cudaError_t launch_local_sum<T>(const Common<T>&, cudaStream_t);           \
  template cudaError_t launch_consensus_metric<T>(const int64_t*, int, int, int, int, double*, double*, double*, cudaStream_t); \
  template cudaError_t launch_dinno_update<T>(const DinnoArgs<T>&, cudaStream_t);     \
  template cudaError_t launch_local_step<T>(const LocalArgs<T>&, cudaStream_t);       \
  template cudaError_t launch_dsgd_mix<T>(const Common<T>&, cudaStream_t);            \
  template cudaError_t launch_dsgd_step<T>(const Common<T>&, cudaStream_t);           \
  template cudaError_t launch_dsgt_init<T>(const DsgtArgs<T>&, cudaStream_t);         \
  template cudaError_t launch_dsgt_mix<T>(const DsgtArgs<T>&, cudaStream_t);          \
  template cudaError_t launch_dsgt_track<T>(const DsgtArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_ed_mix<T>(const EdArgs<T>&, cudaStream_t);              \
  template cudaError_t launch_ed_step<T>(const EdArgs<T>&, cudaStream_t);             \
  template cudaError_t launch_dsgdm_step<T>(const MomentumArgs<T>&, cudaStream_t);    \
  template cudaError_t launch_choco_mix<T>(const ChocoArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_choco_step<T>(const ChocoArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_beer_mix<T>(const BeerArgs<T>&, cudaStream_t);          \
  template cudaError_t launch_beer_step<T>(const BeerArgs<T>&, cudaStream_t);         \
  template cudaError_t launch_kgt_mix<T>(const KgtArgs<T>&, cudaStream_t);            \
  template cudaError_t launch_kgt_step<T>(const KgtArgs<T>&, cudaStream_t);           \
  template cudaError_t launch_ag_gossip<T>(const DetagArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_detag_track<T>(const DetagArgs<T>&, cudaStream_t);      \
  template cudaError_t launch_hsgd_track<T>(const HsgdArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_xg_pull<T>(const XgArgs<T>&, cudaStream_t);             \
  template cudaError_t launch_xg_publish<T>(const XgArgs<T>&, cudaStream_t);          \
  template cudaError_t launch_xg_step<T>(const XgArgs<T>&, cudaStream_t);             \
  template cudaError_t launch_pga_sum<T>(const PgaArgs<T>&, cudaStream_t);            \
  template cudaError_t launch_pga_mix<T>(const PgaArgs<T>&, cudaStream_t);            \
  template cudaError_t launch_slowmo_outer<T>(const SlowmoArgs<T>&, cudaStream_t);    \
  template cudaError_t launch_dp_norm<T>(const DpArgs<T>&, cudaStream_t);             \
  template cudaError_t launch_dp_step<T>(const DpArgs<T>&, cudaStream_t);             \
  template cudaError_t launch_mq_mix<T>(const MoniquaArgs<T>&, cudaStream_t);         \
  template cudaError_t launch_mq_step<T>(const MoniquaArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_sparq_mix<T>(const SparqArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_sparq_step<T>(const SparqArgs<T>&, cudaStream_t);       \
  template cudaError_t launch_sparq_publish<T>(const SparqArgs<T>&, cudaStream_t);    \
  template cudaError_t launch_dadaptive_mix<T>(const DAdaptiveArgs<T>&, cudaStream_t); \
  template cudaError_t launch_dadaptive_step<T>(const DAdaptiveArgs<T>&, cudaStream_t); \
  template cudaError_t launch_relay_mix<T>(const RelayArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_relay_step<T>(const RelayArgs<T>&, cudaStream_t);       \
  template cudaError_t launch_pg_mix<T>(const PgArgs<T>&, cudaStream_t);           \
  template cudaError_t launch_pg_step<T>(const PgArgs<T>&, cudaStream_t);          \
  template cudaError_t launch_cg_dist<T>(const ClipArgs<T>&, cudaStream_t);           \
  template cudaError_t launch_cg_mix<T>(const ClipArgs<T>&, cudaStream_t);            \
  template cudaError_t launch_cg_step<T>(const ClipArgs<T>&, cudaStream_t);           \
  template cudaError_t launch_bridge_mix<T>(const ScreenArgs<T>&, cudaStream_t);      \
  template cudaError_t launch_sgp_mix<T>(const SgpArgs<T>&, cudaStream_t);            \
  template cudaError_t launch_sgp_step<T>(const SgpArgs<T>&, cudaStream_t);           \
  template cudaError_t launch_pdg_mix<T>(const PushDigArgs<T>&, cudaStream_t);        \
  template cudaError_t launch_pdg_track<T>(const PushDigArgs<T>&, cudaStream_t);
NNDT_INST(float)
NNDT_INST(double)

}  // namespace consensus
}  // namespace nndt