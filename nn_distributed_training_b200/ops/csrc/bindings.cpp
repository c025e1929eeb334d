// Python bindings of the sm_90a kernels.  Ops are thin objects that own a filled launch
// struct (raw device addresses supplied by Python, which keeps the tensors alive) and launch on
// PyTorch's current CUDA stream, so they compose with torch.cuda.graph capture: a whole
// consensus round is captured once and replayed.
#include <torch/extension.h>
#include <cstring>
#include <string>
#include <ATen/cuda/CUDAContext.h>
#include <pybind11/pybind11.h>

#include "consensus.h"
#include "mnist.h"
#include "dinno_round.h"

namespace py = pybind11;
using namespace nndt;

static inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
static inline void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
template <typename P> static P* ptr(const py::dict& d, const char* k) {
  if (!d.contains(k) || d[k].is_none()) return nullptr;
  return reinterpret_cast<P*>(d[k].cast<uint64_t>());
}
static int geti(const py::dict& d, const char* k, int dflt = 0) { return d.contains(k) ? d[k].cast<int>() : dflt; }
static double getf(const py::dict& d, const char* k, double dflt = 0) { return d.contains(k) ? d[k].cast<double>() : dflt; }

// ------------------------------------------------------------------ MNIST ----
struct MnistOp {
  mnist::Args a{};
  mnist::GenericShape gs{3, 5, 64, 0, 0.0, 1.0};
  int spb = 8, S = 1, eval_ctas = 1, generic = 0, tc = 0, cl64 = 0;
  alignas(64) unsigned char w1_map[128] = {0};
  explicit MnistOp(const py::dict& d) { update(d); }
  void update(const py::dict& d) {
    a.theta = ptr<const float>(d, "theta"); a.n_pad = geti(d, "n_pad"); a.L = geti(d, "L");
    a.off_wc = geti(d, "off_wc"); a.off_bc = geti(d, "off_bc"); a.off_w1 = geti(d, "off_w1");
    a.off_b1 = geti(d, "off_b1"); a.off_w2 = geti(d, "off_w2"); a.off_b2 = geti(d, "off_b2");
    a.x = ptr<const void>(d, "x"); a.y = ptr<const int64_t>(d, "y");
    a.x_is_u8 = geti(d, "x_is_u8"); a.mean = (float)getf(d, "mean"); a.inv_std = (float)getf(d, "inv_std", 1.0);
    a.direct = geti(d, "direct"); a.batch = geti(d, "batch"); a.seed = geti(d, "seed"); a.node0 = geti(d, "node0");
    a.shard_off = ptr<const int>(d, "shard_off"); a.shard_len = ptr<const int>(d, "shard_len");
    a.calls = ptr<int>(d, "calls"); a.arrive = ptr<unsigned int>(d, "arrive"); a.tune = geti(d, "tune", 1); a.prof = ptr<long long>(d, "step_prof"); a.direct_bs = ptr<const int>(d, "direct_bs");
    a.grad_part = ptr<float>(d, "grad_part"); a.loss_part = ptr<float>(d, "loss_part"); a.loss_mirror = ptr<float>(d, "loss_mirror");
    a.n_val = geti(d, "n_val"); a.val_loss = ptr<float>(d, "val_loss");
    a.val_correct = ptr<unsigned char>(d, "val_correct");
    spb = geti(d, "spb", 8); S = geti(d, "S", 1); eval_ctas = geti(d, "eval_ctas", 1);
    // generic CUDA-core kernel (mnist_generic.cu): any conv shape, fp32 / fp64 (theta, grad_part, val_loss then address doubles)
    generic = geti(d, "generic", 0);
    gs.F = geti(d, "num_filters", 3); gs.KS = geti(d, "kernel_size", 5); gs.LW = geti(d, "linear_width", 64);
    gs.dtype64 = geti(d, "dtype64", 0); gs.mean = getf(d, "mean"); gs.inv_std = getf(d, "inv_std", 1.0);
    // K-split cluster kernel (mnist_tc.cu): needs the W1 tensor map
    cl64 = geti(d, "cl64", 0);
    tc = geti(d, "tc", 0);
    if (tc) {
      const std::string m = d["w1_map"].cast<py::bytes>();
      if (m.size() != 128) throw std::runtime_error("w1_map must be the 128-byte CUtensorMap");
      memcpy(w1_map, m.data(), 128);
    }
  }
  void train() {
    if (cl64) check(mnist::launch_train_cl64(a, gs, S, cur_stream()), "mnist_cl64_train");
    else if (generic) check(mnist::launch_generic_train(a, gs, spb, S, cur_stream()), "convnet_generic_train");
    else if (tc) check(mnist::launch_train_tc(a, w1_map, S, cur_stream()), "mnist_tc_train");
    else check(mnist::launch_train(a, spb, S, cur_stream()), "mnist_train");
  }
  void eval() {
    if (generic) check(mnist::launch_generic_eval(a, gs, eval_ctas, cur_stream()), "convnet_generic_eval");
    else check(mnist::launch_eval(a, eval_ctas, cur_stream()), "mnist_eval");
  }
};

struct GatherOp {
  mnist::GatherArgs a{};
  explicit GatherOp(const py::dict& d) {
    a.x_host = ptr<const unsigned char>(d, "x_host"); a.y_host = ptr<const int64_t>(d, "y_host");
    a.row_bytes = geti(d, "row_bytes"); a.x_stage = ptr<unsigned char>(d, "x_stage");
    a.y_stage = ptr<int64_t>(d, "y_stage"); a.bs_stage = ptr<int>(d, "bs_stage");
    a.P = geti(d, "P"); a.L = geti(d, "L"); a.batch = geti(d, "batch"); a.seed = geti(d, "seed"); a.node0 = geti(d, "node0");
    a.shard_off = ptr<const int>(d, "shard_off"); a.shard_len = ptr<const int>(d, "shard_len");
    a.calls0 = ptr<const int>(d, "calls0"); a.stage_round = ptr<int>(d, "stage_round");
    a.done_ctr = ptr<unsigned int>(d, "done_ctr"); a.max_blocks = geti(d, "max_blocks", 24);
  }
  void launch() { check(mnist::launch_gather(a, cur_stream()), "gather_rows"); }
};

// -------------------------------------------------------------- consensus ----
template <typename T>
static consensus::Common<T> common_from(const py::dict& d) {
  consensus::Common<T> c{};
  c.L = geti(d, "L"); c.n_pad = geti(d, "n_pad"); c.S = geti(d, "S", 1);
  c.theta = ptr<T>(d, "theta"); c.grad_part = ptr<const T>(d, "grad_part");
  c.pub = ptr<T>(d, "pub"); c.C = geti(d, "C", 1); c.pub_L = geti(d, "pub_L", c.L);
  c.nbr_ptr = ptr<const int64_t>(d, "nbr_ptr"); c.nbr_w = ptr<const T>(d, "nbr_w");
  c.self_w = ptr<const T>(d, "self_w"); c.deg = ptr<const int>(d, "deg");
  c.nbr_rank = ptr<const int>(d, "nbr_rank"); c.dmax = geti(d, "dmax");
  c.round_ctr = ptr<int>(d, "round_ctr");
  c.rho = ptr<const T>(d, "rho"); c.lr = ptr<const T>(d, "lr"); c.alpha = ptr<const T>(d, "alpha");
  c.graph_id = ptr<const int>(d, "graph_id");
  c.calls = ptr<int>(d, "calls");
  c.loss_part = ptr<const float>(d, "loss_part"); c.tloss = ptr<float>(d, "tloss");
  c.tdecay = (float)getf(d, "tdecay", 0.0); c.loss_S = geti(d, "loss_S", 1);
  c.flags = ptr<int>(d, "flags"); c.peer_flag = ptr<const int64_t>(d, "peer_flag");
  c.world = geti(d, "world", 1); c.rank = geti(d, "rank", 0);
  c.done_ctr = ptr<unsigned int>(d, "done_ctr"); c.err = ptr<int>(d, "err");
  c.flags_in_kernel = geti(d, "flags_in_kernel", 1);
  c.flag_pull = geti(d, "flag_pull", 0); c.peer_pub = ptr<const int64_t>(d, "peer_pub");
  c.notify_mask = d.contains("notify_mask") ? d["notify_mask"].cast<unsigned long long>() : ~0ull;
  c.node_order = ptr<const int>(d, "node_order");
  c.timeline = ptr<long long>(d, "timeline");
  c.pub_seq = ptr<int>(d, "pub_seq"); c.nbr_seq = ptr<const int64_t>(d, "nbr_seq");
  c.sum_mode = geti(d, "sum_mode", 0); c.n_total = geti(d, "n_total", 0);
  c.sum_local = ptr<double>(d, "sum_local"); c.sum_mc = ptr<const double>(d, "sum_mc");
  c.sum_flags = ptr<int>(d, "sum_flags"); c.peer_sum_flag = ptr<const int64_t>(d, "peer_sum_flag");
  return c;
}

template <typename T>
struct ConsensusOp {
  consensus::Common<T> c{};
  consensus::DinnoArgs<T> dn{};
  consensus::DsgtArgs<T> gt{};
  explicit ConsensusOp(const py::dict& d) {
    c = common_from<T>(d);
    dn.c = c; gt.c = c;
    dn.dual = ptr<T>(d, "dual"); dn.delta = ptr<T>(d, "delta"); dn.m = ptr<T>(d, "m"); dn.v = ptr<T>(d, "v");
    dn.pits = geti(d, "pits", 1); dn.opt = geti(d, "opt", 1); dn.persistent = geti(d, "persistent", 0);
    gt.g_old = ptr<T>(d, "g_old");
  }
  void dinno_update(int step) {
    dn.step = step;
    check(consensus::launch_dinno_update<T>(dn, cur_stream()), "dinno_update");
  }
  void local_sum() { check(consensus::launch_local_sum<T>(c, cur_stream()), "local_sum"); }
  void publish() { check(consensus::launch_publish_round<T>(c, cur_stream()), "publish_round"); }
  void dsgd_mix() { check(consensus::launch_dsgd_mix<T>(c, cur_stream()), "dsgd_mix"); }
  void dsgd_step() { check(consensus::launch_dsgd_step<T>(c, cur_stream()), "dsgd_step"); }
  void dsgt_init() { check(consensus::launch_dsgt_init<T>(gt, cur_stream()), "dsgt_init"); }
  void dsgt_mix() { check(consensus::launch_dsgt_mix<T>(gt, cur_stream()), "dsgt_mix"); }
  void dsgt_track() { check(consensus::launch_dsgt_track<T>(gt, cur_stream()), "dsgt_track"); }
};

template <typename T>
static void bind_consensus(py::module& m, const char* name) {
  py::class_<ConsensusOp<T>>(m, name)
      .def(py::init<const py::dict&>())
      .def("dinno_update", &ConsensusOp<T>::dinno_update)
      .def("local_sum", &ConsensusOp<T>::local_sum)
      .def("publish", &ConsensusOp<T>::publish)
      .def("dsgd_mix", &ConsensusOp<T>::dsgd_mix)
      .def("dsgd_step", &ConsensusOp<T>::dsgd_step)
      .def("dsgt_init", &ConsensusOp<T>::dsgt_init)
      .def("dsgt_mix", &ConsensusOp<T>::dsgt_mix)
      .def("dsgt_track", &ConsensusOp<T>::dsgt_track);
}

// One launch per DiNNO round (dinno_round.cu): mnist dict + consensus dict + per-step batch sources
struct DinnoRoundOp {
  round::RoundArgs a{};
  int S = 1;
  DinnoRoundOp(const py::dict& md, const py::dict& cd, const py::list& steps) {
    MnistOp mo(md);
    ConsensusOp<float> co(cd);
    a.m = mo.a; a.d = co.dn; S = mo.S;
    a.prof = ptr<long long>(md, "prof");
    if ((int)steps.size() != a.d.pits || a.d.pits > round::kMaxSteps) throw std::runtime_error("DinnoRoundOp: bad step list");
    for (int p = 0; p < a.d.pits; ++p) {
      const py::dict sd = steps[p].cast<py::dict>();
      a.x_step[p] = ptr<const void>(sd, "x"); a.y_step[p] = ptr<const int64_t>(sd, "y");
      a.bs_step[p] = ptr<const int>(sd, "direct_bs");
    }
  }
  void launch() { check(round::launch_dinno_round(a, S, cur_stream()), "dinno_round"); }
};

void bind_mlp(py::module& m);     // mlp_bind.cpp
void bind_rl(py::module& m);      // rl_bind.cpp
void bind_runtime(py::module& m); // runtime.cpp

PYBIND11_MODULE(_C, m) {
  m.doc() = "nn_distributed_training_b200 sm_90a kernels";
  py::class_<MnistOp>(m, "MnistOp")
      .def(py::init<const py::dict&>())
      .def("update", &MnistOp::update)
      .def("train", &MnistOp::train)
      .def("eval", &MnistOp::eval);
  py::class_<GatherOp>(m, "GatherOp").def(py::init<const py::dict&>()).def("launch", &GatherOp::launch);
  m.def("debug_batch_indices", [](int mm, int B, int call, int seed, int node, uint64_t out, uint64_t out_size) {
    check(mnist::launch_batch_indices(mm, B, call, seed, node, reinterpret_cast<int*>(out),
                                      reinterpret_cast<int*>(out_size), cur_stream()), "batch_indices");
  });
  m.def("consensus_metric", [](bool f64, uint64_t rows, int N, int n_pad, int local0, int L, uint64_t inv_norm,
                               uint64_t out_pair, uint64_t out_mean) {
    auto r = reinterpret_cast<const int64_t*>(rows);
    auto a = reinterpret_cast<double*>(inv_norm); auto b = reinterpret_cast<double*>(out_pair); auto c = reinterpret_cast<double*>(out_mean);
    check(f64 ? consensus::launch_consensus_metric<double>(r, N, n_pad, local0, L, a, b, c, cur_stream())
              : consensus::launch_consensus_metric<float>(r, N, n_pad, local0, L, a, b, c, cur_stream()), "consensus_metric");
  });
  m.def("convnet_generic_smem_bytes", [](int F, int KS, int LW, int dtype64, int spb) {
    return (size_t)mnist::generic_smem_bytes(mnist::GenericShape{F, KS, LW, dtype64, 0.0, 1.0}, dtype64, spb);
  });
  m.def("make_w1_tensor_map", [](uint64_t theta, int n_pad, int L, int off_w1) {
    unsigned char buf[128];
    check(mnist::make_w1_tensor_map(reinterpret_cast<const float*>(theta), n_pad, L, off_w1, buf), "make_w1_tensor_map");
    return py::bytes(reinterpret_cast<const char*>(buf), 128);
  });
  m.def("mnist_tc_max_clusters", []() { return mnist::tc_max_active_clusters(); });
  m.def("mnist_cl64_max_clusters", [](int nsplit) { return mnist::cl64_max_active_clusters(nsplit); }, py::arg("nsplit") = 1);
  m.def("mnist_cl64_cluster_ctas", []() { return mnist::cl64_cluster_ctas(); });
  m.def("rank_barrier", [](uint64_t slots, uint64_t peer_slot, int world, int rank, int epoch, uint64_t gate, uint64_t err) {
    check(consensus::launch_rank_barrier(reinterpret_cast<int*>(slots), reinterpret_cast<const int64_t*>(peer_slot), world, rank,
                                         epoch, reinterpret_cast<const volatile int*>(gate), reinterpret_cast<int*>(err), cur_stream()),
          "rank_barrier");
  });
  m.def("spin", [](long long cycles) { check(consensus::launch_spin(cycles, cur_stream()), "spin"); });
  py::class_<DinnoRoundOp>(m, "DinnoRoundOp")
      .def(py::init<const py::dict&, const py::dict&, const py::list&>())
      .def("launch", &DinnoRoundOp::launch);
  m.def("dinno_round_max_clusters", [](int S) { return round::max_active_clusters(S); });
  bind_consensus<float>(m, "ConsensusOpF32");
  bind_consensus<double>(m, "ConsensusOpF64");
  bind_mlp(m);
  bind_rl(m);
  bind_runtime(m);
}
