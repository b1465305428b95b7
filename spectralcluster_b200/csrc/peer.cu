// Peer memory over NVLink / NVSwitch for the row-sharded pipeline (one process per GPU):
// CUDA IPC handles make a peer rank's Y planes and S row block addressable from this process, so
//   * the Y row blocks a rank multiplies against are PULLED by the copy engines
//     (sc_memcpy_async on a side stream: no SM is taken away from the persistent GEMM), and
//   * the transposed S blocks are PUSHED by the GEMM epilogue itself (k_gemm_wgmma `mirror`).
// The reference has no counterpart (single process, single thread: SURVEY.md section 1).
#include "common.cuh"

#include <cuda.h>
#include <cstring>
#include <map>
#include <mutex>
#include <string>

namespace sc {

typedef CUresult (*GetRangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);

static GetRangeFn get_range_fn() {
  static GetRangeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<GetRangeFn>(p);
  });
  return fn;
}

// one cudaIpcOpenMemHandle per (handle) and process: a second open of the same allocation fails
static std::mutex g_ipc_lock;
static std::map<std::string, void*> g_ipc_open;

}  // namespace sc

using namespace sc;

extern "C" int sc_ipc_export(sc_context* ctx, const void* dev_ptr, void* handle_out,
                             int64_t* offset_out) {
  SC_REQUIRE(ctx && dev_ptr && handle_out && offset_out, "sc_ipc_export: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  GetRangeFn range = get_range_fn();
  SC_REQUIRE(range != nullptr, "sc_ipc_export: cuMemGetAddressRange is not available");
  CUdeviceptr base = 0;
  size_t size = 0;
  const CUresult r = range(&base, &size, (CUdeviceptr)dev_ptr);
  SC_REQUIRE(r == CUDA_SUCCESS, "sc_ipc_export: cuMemGetAddressRange failed (%d)", (int)r);
  cudaIpcMemHandle_t h;
  SC_CUDA(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base)));
  memcpy(handle_out, &h, sizeof(h));
  *offset_out = (int64_t)((CUdeviceptr)dev_ptr - base);
  return 0;
}

extern "C" int sc_ipc_open(sc_context* ctx, const void* handle, int64_t offset, void** out) {
  SC_REQUIRE(ctx && handle && out && offset >= 0, "sc_ipc_open: bad arguments");
  SC_CUDA(cudaSetDevice(ctx->device));
  const std::string key(reinterpret_cast<const char*>(handle), 64);
  std::lock_guard<std::mutex> guard(g_ipc_lock);
  auto it = g_ipc_open.find(key);
  void* base = nullptr;
  if (it != g_ipc_open.end()) {
    base = it->second;
  } else {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    SC_CUDA(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    g_ipc_open[key] = base;
  }
  *out = static_cast<char*>(base) + offset;
  return 0;
}

extern "C" int sc_ipc_close_all(sc_context* ctx) {
  SC_REQUIRE(ctx, "sc_ipc_close_all: bad arguments");
  std::lock_guard<std::mutex> guard(g_ipc_lock);
  for (auto& kv : g_ipc_open) cudaIpcCloseMemHandle(kv.second);
  g_ipc_open.clear();
  return 0;
}

extern "C" int sc_memcpy_async(sc_context* ctx, void* dst, const void* src, int64_t bytes,
                               void* stream) {
  SC_REQUIRE(ctx && dst && src && bytes >= 0, "sc_memcpy_async: bad arguments");
  SC_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, as_stream(stream)));
  return 0;
}
