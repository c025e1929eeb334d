// CUDA IPC helpers for the peer-mapped symmetric buffers (fallback of parallel/symm.py).
#include <cuda_runtime.h>
#include <pybind11/pybind11.h>

#include <cstring>
#include <stdexcept>
#include <string>

namespace py = pybind11;

static void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void bind_runtime(py::module& m) {
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
