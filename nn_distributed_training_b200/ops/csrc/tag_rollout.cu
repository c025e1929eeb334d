// One launch = one whole multi-agent PPO rollout on the predator-prey environment (rl/simple_tag.py, rl/dist_ppo.py):
// every episode of a batch, every cycle, every predator's actor MLP and Gaussian action, the heuristic prey, the contact
// physics, the shared predator reward and finally the rewards-to-go.
//
// Decomposition: worlds (episode, env) are independent, so a CTA owns `wpb` of them for their whole life; the host picks
// wpb so that even a 16-world batch spreads over 16 SMs.  Each distinct actor is staged once per CTA in shared memory,
// transposed (Wt[k][o]), when it fits; otherwise (float64 with several 64-wide actors) the weights are read in place
// through L1/L2.  In a layer one thread owns an (actor output neuron, predator, group of RW worlds): the weight read is
// conflict free along o and the activation read is a broadcast.  Every sum runs in a fixed order, nothing is atomic,
// so two launches are bitwise equal.
//
// Arithmetic follows the torch path op by op: products that torch rounds before an addition use __*_rn (so no FMA
// contraction), divisions and square roots are correctly rounded despite --use_fast_math, and softplus' exp/log1p are
// evaluated in double.  The MLP itself is plain fp32 (or fp64) FMA.
//
// Noise: Philox4x32-10 keyed by the 64-bit key; the counter names (world, episode, cycle, predator, rollout index), so
// the draws do not depend on the grid.  Box-Muller in double turns 6 words into the 5 standard normals of an action.
#include <curand_philox4x32_x.h>

#include "common.cuh"
#include "tag_rollout.h"

namespace nndt {
namespace tag {

namespace {

constexpr int NT = 256, HW = kMaxWidth;   // threads per CTA, activation row stride

NNDT_DEVINL float add_rn(float x, float y) { return __fadd_rn(x, y); }
NNDT_DEVINL double add_rn(double x, double y) { return __dadd_rn(x, y); }
NNDT_DEVINL float sub_rn(float x, float y) { return __fsub_rn(x, y); }
NNDT_DEVINL double sub_rn(double x, double y) { return __dsub_rn(x, y); }
NNDT_DEVINL float mul_rn(float x, float y) { return __fmul_rn(x, y); }
NNDT_DEVINL double mul_rn(double x, double y) { return __dmul_rn(x, y); }
NNDT_DEVINL float div_rn(float x, float y) { return __fdiv_rn(x, y); }
NNDT_DEVINL double div_rn(double x, double y) { return __ddiv_rn(x, y); }
NNDT_DEVINL float sqrt_rn(float x) { return __fsqrt_rn(x); }
NNDT_DEVINL double sqrt_rn(double x) { return __dsqrt_rn(x); }

template <typename T> NNDT_DEVINL T norm2(T x, T y) { return sqrt_rn(add_rn(mul_rn(x, x), mul_rn(y, y))); }

// torch.nn.functional.softplus with beta 1 and threshold 20
template <typename T> NNDT_DEVINL T softplus(T x) { return x > (T)20 ? x : (T)log1p(exp((double)x)); }

// Contact force on an agent at distance (dx, dy) from a body, dmin = sum of the radii (simple_tag._contact_forces).
template <typename T> NNDT_DEVINL void contact(T dx, T dy, T dmin, T& fx, T& fy) {
  const T k = (T)1e-3;
  const T dist = fmax(norm2(dx, dy), (T)1e-12);
  const T pen = mul_rn(softplus(div_rn(-sub_rn(dist, dmin), k)), k);
  fx = add_rn(fx, mul_rn(div_rn(mul_rn((T)100, dx), dist), pen));
  fy = add_rn(fy, mul_rn(div_rn(mul_rn((T)100, dy), dist), pen));
}

NNDT_DEVINL void box_muller(uint32_t x, uint32_t y, double& z0, double& z1) {
  const double u1 = ((double)x + 0.5) * 2.3283064365386963e-10;   // (0, 1)
  const double u2 = ((double)y + 0.5) * 2.3283064365386963e-10;
  const double r = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi(2.0 * u2, &s, &c);
  z0 = r * c;
  z1 = r * s;
}

__host__ __device__ inline size_t actor_numel(const Args& a) {
  size_t n = 0;
  for (int l = 0; l < a.nl; ++l) n += (size_t)a.dims[l] * a.dims[l + 1] + a.dims[l + 1];
  return n;
}

// Shared memory, in elements of T: staged actors, two activation buffers [wpb][N][HW], world state.
struct Layout {
  size_t w, h0, h1, pos, vel, act, total;
};
__host__ __device__ inline Layout layout(const Args& a, int wpb, int stage) {
  Layout L;
  size_t o = 0;
  L.w = o;   o += stage ? (size_t)a.n_actor * actor_numel(a) : 0;
  L.h0 = o;  o += (size_t)wpb * a.N * HW;
  L.h1 = o;  o += (size_t)wpb * a.N * HW;
  L.pos = o; o += (size_t)wpb * a.A * 2;
  L.vel = o; o += (size_t)wpb * a.A * 2;
  L.act = o; o += (size_t)wpb * a.A * kActDim;
  L.total = o;
  return L;
}

// out[w][i][o] = act(b[o] + sum_k in[w][i][k] W[o][k]) for the RW worlds of a group; the weight is read as
// Wp[k * sk + o * so] (staged transposed: sk = dout, so = 1; in place: sk = 1, so = din).
template <typename T, int RW>
NNDT_DEVINL void neuron(const T* x, T* y, const T* Wp, const T* Bp, int sk, int so, int din, int o, int wstride,
                        bool relu) {
  T acc[RW];
#pragma unroll
  for (int r = 0; r < RW; ++r) acc[r] = (T)0;
  for (int k = 0; k < din; ++k) {
    const T w = Wp[k * sk + o * so];
#pragma unroll
    for (int r = 0; r < RW; ++r) acc[r] = fma(x[r * wstride + k], w, acc[r]);
  }
  const T bb = Bp[o];
#pragma unroll
  for (int r = 0; r < RW; ++r) {
    const T z = acc[r] + bb;
    y[r * wstride + o] = relu ? (z > (T)0 ? z : (T)0) : z;
  }
}

template <typename T, int RW>
__global__ void __launch_bounds__(NT) tag_rollout_kernel(const Args a, const int wpb, const int stage) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sm = reinterpret_cast<T*>(smem_raw);
  const Layout Ly = layout(a, wpb, stage);
  T* sw = sm + Ly.w;
  T* spos = sm + Ly.pos;
  T* svel = sm + Ly.vel;
  T* sact = sm + Ly.act;
  const int tid = threadIdx.x, N = a.N, A = a.A, E = a.E, T_ = a.T, D0 = a.dims[0];
  const int nw = a.n_ep * E, g0 = blockIdx.x * wpb;
  const size_t R = (size_t)a.n_ep * T_ * E;
  const size_t per_actor = actor_numel(a);
  const T* size = reinterpret_cast<const T*>(a.size);
  const T* accel = reinterpret_cast<const T*>(a.accel);
  const T* vmax = reinterpret_cast<const T*>(a.max_speed);
  const T* obst = reinterpret_cast<const T*>(a.obst);
  T* obs_out = reinterpret_cast<T*>(a.obs);
  T* acts_out = reinterpret_cast<T*>(a.acts);
  T* lp_out = reinterpret_cast<T*>(a.log_probs);
  T* rtgs = reinterpret_cast<T*>(a.rtgs);
  T* eps_out = reinterpret_cast<T*>(a.eps);
  T* trace = reinterpret_cast<T*>(a.pos_trace);
  const uint2 key = make_uint2((uint32_t)a.key, (uint32_t)(a.key >> 32));

  if (stage) {
    for (int ac = 0; ac < a.n_actor; ++ac) {
      T* dst = sw + ac * per_actor;
      for (int l = 0; l < a.nl; ++l) {
        const int din = a.dims[l], dout = a.dims[l + 1];
        const T* W = reinterpret_cast<const T*>(a.W[ac][l]);
        const T* B = reinterpret_cast<const T*>(a.b[ac][l]);
        for (int q = tid; q < din * dout; q += NT) {
          const int o = q / din, k = q - o * din;
          dst[k * dout + o] = W[q];
        }
        for (int o = tid; o < dout; o += NT) dst[din * dout + o] = B[o];
        dst += (size_t)din * dout + dout;
      }
    }
  }
  for (int q = tid; q < wpb * A * 2; q += NT) {
    const int g = g0 + q / (A * 2);
    spos[q] = g < nw ? reinterpret_cast<const T*>(a.pos0)[(size_t)g0 * A * 2 + q] : (T)0;
    svel[q] = (T)0;
  }
  T ret_sum = (T)0;   // thread lw < wpb: the world's reward summed over cycles
  __syncthreads();

  for (int c = 0; c < T_; ++c) {
    // ---- adversary observations: own vel, own pos, others' relative positions, prey velocities
    T* h = sm + Ly.h0;
    for (int q = tid; q < wpb * N; q += NT) {
      const int lw = q / N, i = q - lw * N, g = g0 + lw;
      const T* p = spos + lw * A * 2;
      const T* v = svel + lw * A * 2;
      T* x = h + (size_t)q * HW;
      int m = 0;
      x[m++] = v[2 * i]; x[m++] = v[2 * i + 1]; x[m++] = p[2 * i]; x[m++] = p[2 * i + 1];
      for (int j = 0; j < A; ++j) {
        if (j == i) continue;
        x[m++] = sub_rn(p[2 * j], p[2 * i]);
        x[m++] = sub_rn(p[2 * j + 1], p[2 * i + 1]);
      }
      for (int j = N; j < A; ++j) { x[m++] = v[2 * j]; x[m++] = v[2 * j + 1]; }
      if (g < nw) {
        const int ep = g / E, e = g - ep * E;
        T* o = obs_out + ((size_t)i * R + ((size_t)ep * T_ + c) * E + e) * D0;
        for (int k = 0; k < D0; ++k) o[k] = x[k];
      }
    }
    __syncthreads();

    // ---- actor MLPs
    T* in = sm + Ly.h0;
    T* out = sm + Ly.h1;
    size_t woff = 0;
    for (int l = 0; l < a.nl; ++l) {
      const int din = a.dims[l], dout = a.dims[l + 1];
      const bool relu = l + 1 < a.nl;
      const int items = (wpb / RW) * N * dout;
      for (int q = tid; q < items; q += NT) {
        const int o = q % dout, t = q / dout, i = t % N, wg = t / N;
        const int ac = a.actor_of[i];
        const size_t base = ((size_t)wg * RW * N + i) * HW;
        if (stage) {
          const T* Wp = sw + ac * per_actor + woff;
          neuron<T, RW>(in + base, out + base, Wp, Wp + din * dout, dout, 1, din, o, N * HW, relu);
        } else {
          neuron<T, RW>(in + base, out + base, reinterpret_cast<const T*>(a.W[ac][l]),
                        reinterpret_cast<const T*>(a.b[ac][l]), 1, din, din, o, N * HW, relu);
        }
      }
      woff += (size_t)din * dout + dout;
      T* t = in; in = out; out = t;
      __syncthreads();
    }

    // ---- Gaussian predator actions and log-probs; heuristic prey action from prey 0's observation
    for (int q = tid; q < wpb * N + wpb; q += NT) {
      if (q < wpb * N) {
        const int lw = q / N, i = q - lw * N, g = g0 + lw;
        const int ep = g / E, e = g - ep * E;
        const uint32_t cw = ((uint32_t)c << 4) | ((uint32_t)i << 1);
        const uint4 r0 = curand_Philox4x32_10(make_uint4((uint32_t)e, (uint32_t)ep, cw, a.index), key);
        const uint4 r1 = curand_Philox4x32_10(make_uint4((uint32_t)e, (uint32_t)ep, cw | 1u, a.index), key);
        double z[6];
        box_muller(r0.x, r0.y, z[0], z[1]);
        box_muller(r0.z, r0.w, z[2], z[3]);
        box_muller(r1.x, r1.y, z[4], z[5]);
        const T* mean = in + (size_t)q * HW;
        const T std_ = (T)a.noise_std;
        T S = (T)0;
        const size_t row = ((size_t)ep * T_ + c) * E + e;
#pragma unroll
        for (int k = 0; k < kActDim; ++k) {
          const T ek = (T)z[k];
          const T act = add_rn(mean[k], mul_rn(std_, ek));
          const T d = sub_rn(act, mean[k]);
          S = add_rn(S, mul_rn(d, d));
          sact[(lw * A + i) * kActDim + k] = act;
          if (g < nw) {
            acts_out[((size_t)i * R + row) * kActDim + k] = act;
            if (eps_out) eps_out[((size_t)i * R + row) * kActDim + k] = ek;
          }
        }
        if (g < nw) lp_out[(size_t)i * R + row] = sub_rn(div_rn(mul_rn((T)-0.5, S), (T)a.cov_var), (T)a.lp_const);
      } else {
        const int lw = q - wpb * N;
        const T* p = spos + lw * A * 2;
        const T qx = p[2 * N], qy = p[2 * N + 1];
        int near = 0;
        T best = (T)0;
        for (int j = 0; j < N; ++j) {
          const T nrm = norm2(sub_rn(p[2 * j], qx), sub_rn(p[2 * j + 1], qy));
          if (j == 0 || nrm < best) { best = nrm; near = j; }
        }
        const T dx = sub_rn(p[2 * near], qx), dy = sub_rn(p[2 * near + 1], qy);
        const T m = fmax(fmax(fabs(dx), fabs(dy)), (T)1e-12);
        const T fx = div_rn(-dx, m), fy = div_rn(-dy, m);
        T a1 = fmax(fx, (T)0), a2 = fmax(-fx, (T)0), a3 = fmax(fy, (T)0), a4 = fmax(-fy, (T)0);
        if (qx <= (T)-1.2) a2 = (T)0;
        if (qx >= (T)1.2) a1 = (T)0;
        if (qy <= (T)-1.2) a4 = (T)0;
        if (qy >= (T)1.2) a3 = (T)0;
        for (int j = N; j < A; ++j) {
          T* s = sact + (lw * A + j) * kActDim;
          s[0] = (T)0; s[1] = a1; s[2] = a2; s[3] = a3; s[4] = a4;
        }
      }
    }
    __syncthreads();

    // ---- physics: one thread per (world, agent); contact forces from the pre-step state, damping, then the clamp
    T nvx = (T)0, nvy = (T)0, npx = (T)0, npy = (T)0;
    const int lw_a = tid / A, ag = tid - lw_a * A;
    const bool phys = tid < wpb * A;
    if (phys) {
      const T* p = spos + lw_a * A * 2;
      const T* s = sact + (lw_a * A + ag) * kActDim;
      const T px = p[2 * ag], py = p[2 * ag + 1];
      T sx = (T)0, sy = (T)0;
      for (int b = 0; b < A; ++b)
        if (b != ag) contact(sub_rn(px, p[2 * b]), sub_rn(py, p[2 * b + 1]), add_rn(size[ag], size[b]), sx, sy);
      if (a.n_obst) {
        T ox = (T)0, oy = (T)0;
        const T dmin = add_rn(size[ag], (T)0.2);
        for (int o = 0; o < a.n_obst; ++o) contact(sub_rn(px, obst[2 * o]), sub_rn(py, obst[2 * o + 1]), dmin, ox, oy);
        sx = add_rn(sx, ox);
        sy = add_rn(sy, oy);
      }
      const T fx = add_rn(mul_rn(sub_rn(s[1], s[2]), accel[ag]), sx);
      const T fy = add_rn(mul_rn(sub_rn(s[3], s[4]), accel[ag]), sy);
      const T* v = svel + lw_a * A * 2;
      nvx = add_rn(mul_rn(v[2 * ag], (T)0.75), mul_rn(fx, (T)0.1));
      nvy = add_rn(mul_rn(v[2 * ag + 1], (T)0.75), mul_rn(fy, (T)0.1));
      const T speed = norm2(nvx, nvy), ms = vmax[ag];
      if (speed > ms) {
        const T sp = fmax(speed, (T)1e-12);
        nvx = mul_rn(div_rn(nvx, sp), ms);
        nvy = mul_rn(div_rn(nvy, sp), ms);
      }
      npx = add_rn(px, mul_rn(nvx, (T)0.1));
      npy = add_rn(py, mul_rn(nvy, (T)0.1));
    }
    __syncthreads();
    if (phys) {
      svel[tid * 2] = nvx; svel[tid * 2 + 1] = nvy;
      spos[tid * 2] = npx; spos[tid * 2 + 1] = npy;
      const int g = g0 + lw_a;
      if (trace && g < nw) {
        const int ep = g / E, e = g - ep * E;
        T* t = trace + ((((size_t)ep * T_ + c) * E + e) * A + ag) * 2;
        t[0] = npx; t[1] = npy;
      }
    }
    __syncthreads();

    // ---- shared predator reward: -0.1 sum_i min_prey dist + 10 per colliding (predator, prey) pair
    if (tid < wpb && g0 + tid < nw) {
      const T* p = spos + tid * A * 2;
      T sum = (T)0;
      int hits = 0;
      for (int i = 0; i < N; ++i) {
        T mn = (T)0;
        for (int j = N; j < A; ++j) {
          const T d = norm2(sub_rn(p[2 * i], p[2 * j]), sub_rn(p[2 * i + 1], p[2 * j + 1]));
          hits += d < (T)0.125;
          mn = (j == N || d < mn) ? d : mn;
        }
        sum = add_rn(sum, mn);
      }
      const T r = add_rn(mul_rn((T)-0.1, sum), mul_rn((T)10, (T)hits));
      ret_sum = add_rn(ret_sum, r);
      const int g = g0 + tid, ep = g / E, e = g - ep * E;
      rtgs[((size_t)ep * T_ + c) * E + e] = r;   // predator 0's row holds the rewards until the episode ends
    }
  }

  // ---- rewards-to-go, episode return, final state
  if (tid < wpb && g0 + tid < nw) {
    const int g = g0 + tid, ep = g / E, e = g - ep * E;
    const T gamma = (T)a.gamma;
    T run = (T)0;
    for (int c = T_ - 1; c >= 0; --c) {
      const size_t row = ((size_t)ep * T_ + c) * E + e;
      run = add_rn(rtgs[row], mul_rn(gamma, run));
      for (int i = 0; i < N; ++i) rtgs[(size_t)i * R + row] = run;
    }
    T ret = ret_sum;
    for (int i = 1; i < N; ++i) ret = add_rn(ret, ret_sum);
    reinterpret_cast<T*>(a.ep_returns)[g] = ret;
  }
  for (int q = tid; q < wpb * A * 2; q += NT) {
    if (g0 + q / (A * 2) < nw) {
      reinterpret_cast<T*>(a.final_pos)[(size_t)g0 * A * 2 + q] = spos[q];
      reinterpret_cast<T*>(a.final_vel)[(size_t)g0 * A * 2 + q] = svel[q];
    }
  }
}

template <typename T, int RW>
cudaError_t launch_t(const Args& a, const Plan& p, cudaStream_t st) {
  auto kern = tag_rollout_kernel<T, RW>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
  if (e != cudaSuccess) return e;
  const int nw = a.n_ep * a.E;
  kern<<<(nw + p.wpb - 1) / p.wpb, NT, p.smem, st>>>(a, p.wpb, p.stage);
  return cudaGetLastError();
}

}  // namespace

const char* check(const Args& a) {
  if (a.N < 1 || a.n_good < 1 || a.A != a.N + a.n_good || a.A > kMaxAgents) return "needs 1..7 predators, >= 1 prey, <= 8 agents";
  if (a.n_obst < 0 || a.n_obst > kMaxObst) return "needs <= 8 obstacles";
  if (a.nl < 1 || a.nl > kMaxLayers) return "needs an actor with 1..5 linear layers";
  if (a.dims[0] != 4 + 2 * (a.A - 1) + 2 * a.n_good) return "actor input width != adversary observation width";
  if (a.dims[a.nl] != kActDim) return "actor output width != 5";
  for (int l = 0; l <= a.nl; ++l)
    if (a.dims[l] < 1 || a.dims[l] > kMaxWidth) return "actor widths must be 1..64";
  if (a.n_actor < 1 || a.n_actor > a.N) return "needs 1..N actors";
  for (int i = 0; i < a.N; ++i) {
    if (a.actor_of[i] < 0 || a.actor_of[i] >= a.n_actor) return "bad actor index";
  }
  for (int ac = 0; ac < a.n_actor; ++ac)
    for (int l = 0; l < a.nl; ++l)
      if (!a.W[ac][l] || !a.b[ac][l]) return "missing actor parameter";
  if (a.E < 1 || a.n_ep < 1 || a.T < 1 || a.T >= (1 << 27)) return "needs E, n_ep >= 1 and 1 <= T < 2^27";
  if (!a.pos0 || !a.size || !a.accel || !a.max_speed || (a.n_obst && !a.obst) || !a.obs || !a.acts || !a.log_probs ||
      !a.rtgs || !a.ep_returns || !a.final_pos || !a.final_vel)
    return "missing buffer";
  return nullptr;
}

Plan plan(const Args& a) {
  int dev = 0, nsm = 132, optin = 227 * 1024;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  const size_t es = a.dtype64 ? sizeof(double) : sizeof(float);
  const int nw = a.n_ep * a.E;
  int wpb = (nw + nsm - 1) / nsm;
  if (wpb > NT / a.A) wpb = NT / a.A;   // the physics step runs one thread per (world, agent)
  if (wpb >= 4) wpb &= ~3;             // multiples of 4 take the 4-world register blocking
  auto bytes = [&](int w, int s) { return layout(a, w, s).total * es; };
  int stage = bytes(wpb, 1) <= (size_t)optin;
  while (!stage && wpb > 1 && bytes(wpb, 0) > (size_t)optin) wpb = wpb > 4 ? wpb - 4 : wpb - 1;
  return Plan{wpb, stage, bytes(wpb, stage)};
}

cudaError_t launch(const Args& a, cudaStream_t st) {
  if (check(a)) return cudaErrorInvalidValue;
  const Plan p = plan(a);
  if (a.dtype64) return p.wpb % 4 == 0 ? launch_t<double, 4>(a, p, st) : launch_t<double, 1>(a, p, st);
  return p.wpb % 4 == 0 ? launch_t<float, 4>(a, p, st) : launch_t<float, 1>(a, p, st);
}

}  // namespace tag
}  // namespace nndt
