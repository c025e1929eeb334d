// Native runtime pieces around the kernels:
//  * HostBatchLoader — multi-threaded minibatch assembler for the host-fed ("end-to-end")
//    input pipeline: worker threads gather the rows of upcoming rounds (same stateless sampler
//    as the device path) into a ring of pinned staging slots ahead of the consumer, which only
//    issues one H2D copy per round.  Replaces the reference's Python DataLoader
//    (problems/dist_mnist_problem.py:45-54,83-98) on that path.
//  * CUDA IPC helpers for the peer-mapped symmetric buffers (fallback of parallel/symm.py).
#include <cuda_runtime.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <atomic>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "sampler_host.h"

namespace py = pybind11;
using namespace nndt::host;

class HostBatchLoader {
 public:
  HostBatchLoader(uint64_t x, uint64_t y, int row_bytes, std::vector<int> shard_off, std::vector<int> shard_len,
                  std::vector<int64_t> calls0, int batch, int steps_per_round, int seed, int node0,
                  std::vector<uint64_t> slot_x, std::vector<uint64_t> slot_y, std::vector<uint64_t> slot_bs,
                  int n_threads)
      : x_(reinterpret_cast<const uint8_t*>(x)), y_(reinterpret_cast<const int64_t*>(y)), row_(row_bytes),
        off_(std::move(shard_off)), len_(std::move(shard_len)), calls0_(std::move(calls0)), B_(batch),
        P_(steps_per_round), seed_(seed), node0_(node0), sx_(std::move(slot_x)), sy_(std::move(slot_y)),
        sb_(std::move(slot_bs)) {
    L_ = (int)off_.size();
    nslots_ = (int)sx_.size();
    state_.assign(nslots_, kEmpty);
    round_of_.assign(nslots_, -1);
    for (int t = 0; t < std::max(1, n_threads); ++t) workers_.emplace_back([this] { work(); });
  }
  ~HostBatchLoader() { stop(); }

  void stop() {
    {
      std::lock_guard<std::mutex> g(mu_);
      if (stop_) return;
      stop_ = true;
    }
    cv_.notify_all();
    for (auto& w : workers_) if (w.joinable()) w.join();
  }

  // slot holding the batches of the next round to consume (blocks until assembled)
  int acquire() {
    py::gil_scoped_release rel;
    return acquire_nogil();
  }
  int acquire_nogil() {
    std::unique_lock<std::mutex> lk(mu_);
    const int64_t want = next_consume_;
    const int slot = (int)(want % nslots_);
    cv_.wait(lk, [&] { return stop_ || (state_[slot] == kReady && round_of_[slot] == want); });
    if (stop_) throw std::runtime_error("loader stopped");
    state_[slot] = kInUse;
    ++next_consume_;
    return slot;
  }
  // the consumer's H2D copy out of `slot` has completed
  void release(int slot) {
    {
      std::lock_guard<std::mutex> g(mu_);
      state_[slot] = kEmpty;
    }
    cv_.notify_all();
  }
  int64_t rounds_assembled() const { return next_fill_.load(); }

 private:
  enum { kEmpty = 0, kFilling = 1, kReady = 2, kInUse = 3 };

  void work() {
    for (;;) {
      int64_t round; int slot;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return stop_ || state_[(int)(next_fill_ % nslots_)] == kEmpty; });
        if (stop_) return;
        round = next_fill_++;
        slot = (int)(round % nslots_);
        state_[slot] = kFilling;
      }
      fill(slot, round);
      {
        std::lock_guard<std::mutex> g(mu_);
        round_of_[slot] = round;
        state_[slot] = kReady;
      }
      cv_.notify_all();
    }
  }

  void fill(int slot, int64_t round) {
    uint8_t* xs = reinterpret_cast<uint8_t*>(sx_[slot]);
    int64_t* ys = reinterpret_cast<int64_t*>(sy_[slot]);
    int32_t* bs = reinterpret_cast<int32_t*>(sb_[slot]);
    for (int p = 0; p < P_; ++p) {
      for (int l = 0; l < L_; ++l) {
        const uint32_t m = (uint32_t)len_[l];
        const BatchLoc loc = locate_batch((uint32_t)(calls0_[l] + round * P_ + p), m, (uint32_t)B_);
        const uint32_t key = mix_key((uint32_t)seed_, (uint32_t)(node0_ + l), loc.epoch);
        uint8_t* xd = xs + ((size_t)(p * L_ + l) * B_) * row_;
        int64_t* yd = ys + (size_t)(p * L_ + l) * B_;
        bs[p * L_ + l] = (int32_t)loc.size;
        for (uint32_t t = 0; t < loc.size; ++t) {
          const size_t src = (size_t)off_[l] + feistel_permute(loc.start + t, m, key);
          std::memcpy(xd + (size_t)t * row_, x_ + src * row_, row_);
          yd[t] = y_[src];
        }
      }
    }
  }

  const uint8_t* x_; const int64_t* y_; int row_;
  std::vector<int> off_, len_; std::vector<int64_t> calls0_;
  int B_, P_, seed_, node0_, L_ = 0, nslots_ = 0;
  std::vector<uint64_t> sx_, sy_, sb_;
  std::vector<int> state_; std::vector<int64_t> round_of_;
  std::mutex mu_; std::condition_variable cv_;
  std::atomic<int64_t> next_fill_{0};
  int64_t next_consume_ = 0;
  bool stop_ = false;
  std::vector<std::thread> workers_;
};

static void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

// Native per-round driver of the host-fed pipeline.  Round r uses device staging set (r & 1):
//   copy stream   : wait(consumed[b]) -> H2D x/y/bs from the loader's pinned slot -> record(copied[b])
//                   -> host callback releases the slot back to the loader threads
//   compute stream: wait(copied[b]) -> launch the captured round graph of set b (kernels + D2H loss)
//                   -> record(consumed[b])
// so the H2D copy of round r+1 overlaps the kernels of round r and Python is out of the loop.
class HostFedRunner {
 public:
  struct Copy { uint64_t dst, src_off; size_t bytes; };
  HostFedRunner(HostBatchLoader* loader, std::vector<uint64_t> graph_execs, uint64_t compute_stream,
                std::vector<uint64_t> slot_x, std::vector<uint64_t> slot_y, std::vector<uint64_t> slot_bs,
                std::vector<uint64_t> stage_x, std::vector<uint64_t> stage_y, std::vector<uint64_t> stage_bs,
                size_t x_bytes, size_t y_bytes, size_t bs_bytes)
      : loader_(loader), execs_(std::move(graph_execs)), compute_(reinterpret_cast<cudaStream_t>(compute_stream)),
        sx_(std::move(slot_x)), sy_(std::move(slot_y)), sb_(std::move(slot_bs)), dx_(std::move(stage_x)),
        dy_(std::move(stage_y)), db_(std::move(stage_bs)), xb_(x_bytes), yb_(y_bytes), bb_(bs_bytes) {
    cuda_check(cudaStreamCreateWithFlags(&copy_, cudaStreamNonBlocking), "cudaStreamCreate");
    for (int b = 0; b < 2; ++b) {
      cuda_check(cudaEventCreateWithFlags(&copied_[b], cudaEventDisableTiming), "cudaEventCreate");
      cuda_check(cudaEventCreateWithFlags(&consumed_[b], cudaEventDisableTiming), "cudaEventCreate");
    }
  }
  ~HostFedRunner() {
    cudaStreamSynchronize(copy_);
    for (int b = 0; b < 2; ++b) { cudaEventDestroy(copied_[b]); cudaEventDestroy(consumed_[b]); }
    cudaStreamDestroy(copy_);
  }

  void run(int rounds) {
    py::gil_scoped_release rel;
    for (int i = 0; i < rounds; ++i, ++round_) {
      const int b = (int)(round_ & 1);
      const int slot = loader_->acquire_nogil();
      if (round_ >= 2) cuda_check(cudaStreamWaitEvent(copy_, consumed_[b], 0), "wait consumed");
      cuda_check(cudaMemcpyAsync(reinterpret_cast<void*>(dx_[b]), reinterpret_cast<void*>(sx_[slot]), xb_, cudaMemcpyHostToDevice, copy_), "h2d x");
      cuda_check(cudaMemcpyAsync(reinterpret_cast<void*>(dy_[b]), reinterpret_cast<void*>(sy_[slot]), yb_, cudaMemcpyHostToDevice, copy_), "h2d y");
      cuda_check(cudaMemcpyAsync(reinterpret_cast<void*>(db_[b]), reinterpret_cast<void*>(sb_[slot]), bb_, cudaMemcpyHostToDevice, copy_), "h2d bs");
      cuda_check(cudaEventRecord(copied_[b], copy_), "record copied");
      auto* rel_arg = new std::pair<HostBatchLoader*, int>(loader_, slot);
      cuda_check(cudaLaunchHostFunc(copy_, &HostFedRunner::release_cb, rel_arg), "host func");
      cuda_check(cudaStreamWaitEvent(compute_, copied_[b], 0), "wait copied");
      cuda_check(cudaGraphLaunch(reinterpret_cast<cudaGraphExec_t>(execs_[b]), compute_), "graph launch");
      cuda_check(cudaEventRecord(consumed_[b], compute_), "record consumed");
    }
  }
  int64_t rounds_done() const { return round_; }

 private:
  static void CUDART_CB release_cb(void* p) {
    auto* a = static_cast<std::pair<HostBatchLoader*, int>*>(p);
    a->first->release(a->second);
    delete a;
  }
  HostBatchLoader* loader_;
  std::vector<uint64_t> execs_;
  cudaStream_t compute_, copy_ = nullptr;
  std::vector<uint64_t> sx_, sy_, sb_, dx_, dy_, db_;
  size_t xb_, yb_, bb_;
  cudaEvent_t copied_[2], consumed_[2];
  int64_t round_ = 0;
};

void bind_runtime(py::module& m) {
  py::class_<HostBatchLoader>(m, "HostBatchLoader")
      .def(py::init<uint64_t, uint64_t, int, std::vector<int>, std::vector<int>, std::vector<int64_t>, int, int, int,
                    int, std::vector<uint64_t>, std::vector<uint64_t>, std::vector<uint64_t>, int>())
      .def("acquire", &HostBatchLoader::acquire)
      .def("release", &HostBatchLoader::release)
      .def("stop", &HostBatchLoader::stop)
      .def("rounds_assembled", &HostBatchLoader::rounds_assembled);
  py::class_<HostFedRunner>(m, "HostFedRunner")
      .def(py::init<HostBatchLoader*, std::vector<uint64_t>, uint64_t, std::vector<uint64_t>, std::vector<uint64_t>,
                    std::vector<uint64_t>, std::vector<uint64_t>, std::vector<uint64_t>, std::vector<uint64_t>, size_t,
                    size_t, size_t>(), py::keep_alive<1, 2>())
      .def("run", &HostFedRunner::run)
      .def("rounds_done", &HostFedRunner::rounds_done);

  // ---- CUDA IPC (legacy handles) for peer mapping of caching-allocator blocks ------------
  m.def("ipc_get_handle", [](uint64_t ptr) {
    void* base = nullptr; size_t size = 0;
    cudaIpcMemHandle_t h;
    // the handle names the whole cudaMalloc allocation: report the offset of ptr inside it
    cuda_check(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(ptr)), "cudaIpcGetMemHandle");
    cudaPointerAttributes at;
    cuda_check(cudaPointerGetAttributes(&at, reinterpret_cast<void*>(ptr)), "cudaPointerGetAttributes");
    (void)base; (void)size;
    // offset within allocation: query via driver-free trick — cudaMemGetAddressRange is driver API,
    // so allocate IPC buffers with a dedicated cudaMalloc (ipc_alloc) to keep offset == 0.
    return py::make_tuple(py::bytes(reinterpret_cast<const char*>(&h), sizeof(h)), (uint64_t)0);
  });
  m.def("ipc_alloc", [](uint64_t nbytes) {
    void* p = nullptr;
    cuda_check(cudaMalloc(&p, nbytes), "cudaMalloc");
    cuda_check(cudaMemset(p, 0, nbytes), "cudaMemset");
    return (uint64_t)p;
  });
  m.def("ipc_open_handle", [](py::bytes hb) {
    std::string s = hb;
    if (s.size() != sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("bad ipc handle");
    cudaIpcMemHandle_t h;
    std::memcpy(&h, s.data(), sizeof(h));
    void* p = nullptr;
    cuda_check(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
    return (uint64_t)p;
  });
  m.def("ipc_close_handle", [](uint64_t p) { cudaIpcCloseMemHandle(reinterpret_cast<void*>(p)); });
  m.def("cuda_free", [](uint64_t p) { cudaFree(reinterpret_cast<void*>(p)); });
}
