// Output stitch over NVLink / NVSwitch PEER MEMORY (clips shard across ranks, the only exchange is the
// all-gather of the output frames).  Every rank owns a landing buffer allocated here, exports it with a CUDA IPC handle,
// and PUSHES its block of frames into every peer's landing buffer with DMA copies on a side stream — copy engines, no SMs.
// Why not NCCL for the payload: an NCCL kernel holds SMs for as long as it runs (and spins on them while it waits for
// the slowest rank), and the kernels of the next forward are persistent, one CTA per SM with static tile striding — a CTA
// that cannot be placed starts only when another one exits.  The ordering flags are therefore 32-bit words in the same
// peer memory, written and awaited by STREAM MEMORY OPERATIONS (cuStreamWriteValue32 / cuStreamWaitValue32: executed by
// the GPU front end, no kernel), so the exchange does not depend on spare SMs.  NCCL / torch.distributed stay for the plumbing
// (process group, exchange of the IPC handles).  Host side: e2fgvi_b200/clips.py (PeerStitcher).
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstring>

#include "launch.h"

namespace e2f {
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the C ABI carries IPC handles as 64 opaque bytes");

using WriteValueFn = CUresult (*)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
using WaitValueFn = CUresult (*)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
using MemsetD32Fn = CUresult (*)(CUdeviceptr, unsigned int, size_t, CUstream);

static void* driver_fn(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
  return p;
}
}  // namespace e2f

extern "C" {

// cudaMalloc'd landing buffer (NOT from a caching allocator: an IPC handle names a whole allocation) + its IPC handle
int e2f_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64) {
  if (!ptr || !handle64 || bytes == 0) {
    e2f::set_error("e2f_peer_alloc: null argument or zero size");
    return -1;
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    e2f::set_error("e2f_peer_alloc: cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  e = cudaMemset(p, 0, bytes);                       // flag words start at 0; the landing zone is deterministic
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    e2f::set_error("e2f_peer_alloc: memset / cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  std::memcpy(handle64, &h, 64);
  *ptr = p;
  return 0;
}

// map a peer rank's landing buffer into this process (enables peer access between the two devices on first use)
int e2f_peer_open(const unsigned char* handle64, void** ptr) {
  if (!ptr || !handle64) {
    e2f::set_error("e2f_peer_open: null argument");
    return -1;
  }
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle64, 64);
  void* p = nullptr;
  const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    e2f::set_error("e2f_peer_open: cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  *ptr = p;
  return 0;
}

int e2f_peer_close(void* ptr) { return ptr ? static_cast<int>(cudaIpcCloseMemHandle(ptr)) : 0; }

int e2f_peer_free(void* ptr) { return ptr ? static_cast<int>(cudaFree(ptr)) : 0; }

// one block of frames -> a (local or peer) landing buffer: a DMA copy on `stream` (unified addressing picks the route)
int e2f_peer_copy(void* dst, const void* src, size_t bytes, void* stream) {
  if (bytes == 0) return 0;
  if (!dst || !src) {
    e2f::set_error("e2f_peer_copy: null pointer");
    return -1;
  }
  const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) e2f::set_error("e2f_peer_copy: cudaMemcpyAsync failed: %s", cudaGetErrorString(e));
  return static_cast<int>(e);
}

// flag word (local or peer) := value, ordered after everything already enqueued on `stream` (no kernel, no SM)
int e2f_peer_signal(void* flag, unsigned int value, void* stream) {
  static const auto fn = reinterpret_cast<e2f::WriteValueFn>(e2f::driver_fn("cuStreamWriteValue32"));
  if (!fn || !flag) {
    e2f::set_error("e2f_peer_signal: cuStreamWriteValue32 unavailable or null flag");
    return -4;
  }
  static std::atomic<int> use_memset{0};             // a driver that refuses the write on peer-mapped memory: 4-byte memset
  CUresult r = CUDA_ERROR_NOT_SUPPORTED;
  if (!use_memset.load(std::memory_order_relaxed))
    r = fn(static_cast<CUstream>(stream), reinterpret_cast<CUdeviceptr>(flag), value, CU_STREAM_WRITE_VALUE_DEFAULT);
  if (r != CUDA_SUCCESS) {
    static const auto ms = reinterpret_cast<e2f::MemsetD32Fn>(e2f::driver_fn("cuMemsetD32Async"));
    const CUresult r2 = ms ? ms(reinterpret_cast<CUdeviceptr>(flag), value, 1, static_cast<CUstream>(stream)) : r;
    if (r2 == CUDA_SUCCESS) {
      use_memset.store(1, std::memory_order_relaxed);
      return 0;
    }
    e2f::set_error("e2f_peer_signal: cuStreamWriteValue32 failed (%d), cuMemsetD32Async failed (%d)", static_cast<int>(r),
                   static_cast<int>(r2));
  }
  return static_cast<int>(r);
}

// `stream` stalls until (int32)(*flag - value) >= 0; `flag` is a word of THIS rank's flag block (peers write it)
int e2f_peer_wait(void* flag, unsigned int value, void* stream) {
  static const auto fn = reinterpret_cast<e2f::WaitValueFn>(e2f::driver_fn("cuStreamWaitValue32"));
  if (!fn || !flag) {
    e2f::set_error("e2f_peer_wait: cuStreamWaitValue32 unavailable or null flag");
    return -4;
  }
  const CUresult r = fn(static_cast<CUstream>(stream), reinterpret_cast<CUdeviceptr>(flag), value, CU_STREAM_WAIT_VALUE_GEQ);
  if (r != CUDA_SUCCESS) e2f::set_error("e2f_peer_wait: cuStreamWaitValue32 failed (%d)", static_cast<int>(r));
  return static_cast<int>(r);
}

}  // extern "C"
