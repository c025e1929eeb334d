// Binding of the fused predator-prey rollout (tag_rollout.cu).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <stdexcept>
#include <string>

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
  a.eps = mptr(d, "eps"); a.pos_trace = mptr(d, "pos_trace");
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
}
