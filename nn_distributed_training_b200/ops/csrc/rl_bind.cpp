// Bindings of the fused predator-prey rollout (tag_rollout.cu) and of the PPO update kernels (ppo_update.cu).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <stdexcept>
#include <string>

#include "ppo_update.h"
#include "tag_rollout.h"

namespace py = pybind11;
using namespace nndt;

namespace {
const void* cptr(const py::dict& d, const char* k) {
  if (!d.contains(k) || d[k].is_none()) return nullptr;
  return reinterpret_cast<const void*>(d[k].cast<uint64_t>());
}
void* mptr(const py::dict& d, const char* k) { return const_cast<void*>(cptr(d, k)); }

tag::Args tag_args(const py::dict& d) {
  tag::Args a{};
  a.dtype64 = d["dtype64"].cast<int>();
  auto dims = d["dims"].cast<std::vector<int>>();
  auto actor_of = d["actor_of"].cast<std::vector<int>>();
  auto W = d["W"].cast<std::vector<std::vector<uint64_t>>>();
  auto b = d["b"].cast<std::vector<std::vector<uint64_t>>>();
  a.nl = (int)dims.size() - 1;
  a.n_actor = (int)W.size();
  a.N = d["N"].cast<int>();
  if (a.nl < 1 || a.nl > tag::kMaxLayers || a.N < 1 || a.N > tag::kMaxPred || (int)actor_of.size() != a.N ||
      a.n_actor < 1 || a.n_actor > tag::kMaxPred || (int)b.size() != a.n_actor)
    throw std::runtime_error("tag_rollout: bad actor description");
  for (int l = 0; l <= a.nl; ++l) a.dims[l] = dims[l];
  for (int i = 0; i < a.N; ++i) a.actor_of[i] = actor_of[i];
  for (int ac = 0; ac < a.n_actor; ++ac) {
    if ((int)W[ac].size() != a.nl || (int)b[ac].size() != a.nl) throw std::runtime_error("tag_rollout: bad actor description");
    for (int l = 0; l < a.nl; ++l) {
      a.W[ac][l] = reinterpret_cast<const void*>(W[ac][l]);
      a.b[ac][l] = reinterpret_cast<const void*>(b[ac][l]);
    }
  }
  a.n_good = d["n_good"].cast<int>(); a.A = d["A"].cast<int>(); a.n_obst = d["n_obst"].cast<int>();
  a.size = cptr(d, "size"); a.accel = cptr(d, "accel"); a.max_speed = cptr(d, "max_speed"); a.obst = cptr(d, "obst");
  a.E = d["E"].cast<int>(); a.n_ep = d["n_ep"].cast<int>(); a.T = d["T"].cast<int>();
  a.pos0 = cptr(d, "pos0");
  a.gamma = d["gamma"].cast<double>(); a.cov_var = d["cov_var"].cast<double>();
  a.noise_std = d["noise_std"].cast<double>(); a.lp_const = d["lp_const"].cast<double>();
  a.key = d["key"].cast<uint64_t>(); a.index = d["index"].cast<uint32_t>();
  a.obs = mptr(d, "obs"); a.acts = mptr(d, "acts"); a.log_probs = mptr(d, "log_probs"); a.rtgs = mptr(d, "rtgs");
  a.ep_returns = mptr(d, "ep_returns"); a.final_pos = mptr(d, "final_pos"); a.final_vel = mptr(d, "final_vel");
  a.eps = mptr(d, "eps"); a.pos_trace = mptr(d, "pos_trace"); a.rews = mptr(d, "rews");
  return a;
}

// W / b / gW / gb: [N][2][nl] pointers (gW / gb may be absent for the advantage pass).
ppo::Args ppo_args(const py::dict& d) {
  ppo::Args a{};
  a.dtype64 = d["dtype64"].cast<int>();
  a.N = d["N"].cast<int>();
  a.R = d["R"].cast<int>();
  auto dims = d["dims"].cast<std::vector<std::vector<int>>>();
  if (a.N < 1 || a.N > ppo::kMaxNodes || dims.size() != 2) throw std::runtime_error("ppo_update: bad network description");
  for (int n = 0; n < 2; ++n) {
    a.nl[n] = dims[n].empty() ? 0 : (int)dims[n].size() - 1;   // no actor: the advantage pass
    if (a.nl[n] > ppo::kMaxLayers || (a.nl[n] < 1 && (n == ppo::kCritic || !dims[n].empty())))
      throw std::runtime_error("ppo_update: bad network description");
    for (int l = 0; l < (int)dims[n].size(); ++l) a.dims[n][l] = dims[n][l];
  }
  using P3 = std::vector<std::vector<std::vector<uint64_t>>>;
  auto table = [&](const char* k, bool required) {
    P3 t;
    if (d.contains(k) && !d[k].is_none()) t = d[k].cast<P3>();
    else if (required) throw std::runtime_error(std::string("ppo_update: missing ") + k);
    if (!t.empty() && (int)t.size() != a.N) throw std::runtime_error("ppo_update: bad network description");
    for (auto& node : t) {
      if (node.size() != 2) throw std::runtime_error("ppo_update: bad network description");
      for (int n = 0; n < 2; ++n)
        if ((int)node[n].size() != a.nl[n]) throw std::runtime_error("ppo_update: bad network description");
    }
    return t;
  };
  const P3 W = table("W", true), b = table("b", true), gW = table("gW", false), gb = table("gb", false);
  for (int i = 0; i < a.N; ++i)
    for (int n = 0; n < 2; ++n)
      for (int l = 0; l < a.nl[n]; ++l) {
        a.net[i][n].W[l] = reinterpret_cast<const void*>(W[i][n][l]);
        a.net[i][n].b[l] = reinterpret_cast<const void*>(b[i][n][l]);
        a.net[i][n].gW[l] = gW.empty() ? nullptr : reinterpret_cast<void*>(gW[i][n][l]);
        a.net[i][n].gb[l] = gb.empty() ? nullptr : reinterpret_cast<void*>(gb[i][n][l]);
      }
  a.obs = cptr(d, "obs"); a.acts = cptr(d, "acts"); a.old_lp = cptr(d, "old_lp"); a.rtgs = cptr(d, "rtgs");
  a.adv = mptr(d, "adv");
  a.clip = d["clip"].cast<double>(); a.cov_var = d["cov_var"].cast<double>(); a.lp_const = d["lp_const"].cast<double>();
  a.losses = mptr(d, "losses");
  a.nonfinite = reinterpret_cast<int*>(mptr(d, "nonfinite"));
  if (d.contains("gae") && d["gae"].cast<bool>()) {   // GAE(lambda) of the advantage pass
    a.gae = 1;
    a.T = d["T"].cast<int>(); a.E = d["E"].cast<int>();
    a.gamma = d["gamma"].cast<double>(); a.lam = d["lam"].cast<double>();
    a.rews = cptr(d, "rews"); a.returns = mptr(d, "returns"); a.values = mptr(d, "values");
  }
  return a;
}
}  // namespace

void bind_rl(py::module& m) {
  m.def("tag_rollout", [](const py::dict& d) {
    const tag::Args a = tag_args(d);
    if (const char* why = tag::check(a)) throw std::runtime_error(std::string("tag_rollout: ") + why);
    const cudaError_t e = tag::launch(a, at::cuda::getCurrentCUDAStream().stream());
    if (e != cudaSuccess) throw std::runtime_error(std::string("tag_rollout: ") + cudaGetErrorString(e));
  });
  // The plan tag_rollout would launch with on the current device: (worlds per CTA, actors staged, RW, shared memory).
  // Only the shapes of the description are read; its buffers may be absent.
  m.def("tag_rollout_plan", [](const py::dict& d) {
    const tag::Plan p = tag::plan(tag_args(d));
    return py::make_tuple(p.wpb, p.stage, p.rw, p.smem);
  });
  // The plan of ppo_grads (backward) or ppo_advantages on the current device: (rows per tile, chunks per network,
  // dynamic shared memory, workspace bytes of ppo_grads).  Only the shapes of the description are read.
  m.def("ppo_plan", [](const py::dict& d, bool backward) {
    const ppo::Args a = ppo_args(d);
    if (backward && a.nl[ppo::kActor] < 1) throw std::runtime_error("ppo_plan: the gradient pass needs an actor");
    const ppo::Plan p = ppo::plan(a, backward);
    if (p.err != cudaSuccess) throw std::runtime_error(std::string("ppo_plan: ") + cudaGetErrorString(p.err));
    return py::make_tuple(p.tm, p.chunks, p.smem, p.work_bytes);
  });
  m.def("ppo_grads", [](const py::dict& d) {
    const ppo::Args a = ppo_args(d);
    if (const char* why = ppo::check(a, true)) throw std::runtime_error(std::string("ppo_grads: ") + why);
    const ppo::Plan p = ppo::plan(a, true);
    if (p.err != cudaSuccess) throw std::runtime_error(std::string("ppo_grads: ") + cudaGetErrorString(p.err));
    // partial slots: the caller's workspace, or one from the caching allocator on the current device and stream
    void* wp = mptr(d, "work");
    at::Tensor work;
    if (wp) {
      if (d["work_bytes"].cast<uint64_t>() < p.work_bytes) throw std::runtime_error("ppo_grads: workspace too small");
    } else {
      work = at::empty({(int64_t)p.work_bytes}, at::TensorOptions().dtype(at::kByte).device(at::kCUDA));
      wp = work.data_ptr();
    }
    const cudaError_t e = ppo::grads(a, p, wp, at::cuda::getCurrentCUDAStream().stream());
    if (e != cudaSuccess) throw std::runtime_error(std::string("ppo_grads: ") + cudaGetErrorString(e));
  });
  m.def("ppo_advantages", [](const py::dict& d) {
    const ppo::Args a = ppo_args(d);
    if (const char* why = ppo::check(a, false)) throw std::runtime_error(std::string("ppo_advantages: ") + why);
    const cudaError_t e = ppo::advantages(a, at::cuda::getCurrentCUDAStream().stream());
    if (e != cudaSuccess) throw std::runtime_error(std::string("ppo_advantages: ") + cudaGetErrorString(e));
  });
}
