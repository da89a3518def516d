// The deterministic scatter of the sampling backwards (dcn_grad.cu, flow_warp_grad.cu): a kernel writes one
// (destination key, source index) pair per term and the term's coefficient, CUB's stable radix sort orders the pairs by
// destination (each destination's run stays in source order), and a gather kernel adds every destination's run in that
// order.  This header holds what both share on the host: the workspace layout and the sort call with its scratch check.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cstdint>
#include "launch.h"

namespace e2f {
namespace scatter {

constexpr long long SORT_RESERVE_MIN = 65536;   // bytes of sort scratch besides one byte per list entry

// workspace (32-bit elements) of an L-entry list: keys x 2, source indices x 2 (the sort's double buffers),
// coefficients, then the sort scratch, 256-byte aligned
struct Work {
  uint32_t *keys0, *keys1, *vals0, *vals1;
  float* coef;
  void* temp;
  size_t temp_bytes;
};

inline long long body_elems(long long L) { return (5 * L + 63) / 64 * 64; }
inline long long temp_elems(long long L) { return (L + SORT_RESERVE_MIN + 255) / 256 * 64; }
inline long long work_elems(long long L) { return body_elems(L) + temp_elems(L); }

inline Work carve(void* work, long long L) {
  uint32_t* w = static_cast<uint32_t*>(work);
  return Work{w, w + L, w + 2 * L, w + 3 * L, reinterpret_cast<float*>(w + 4 * L), w + body_elems(L),
              static_cast<size_t>(temp_elems(L)) * 4};
}

// Sorts the L pairs of `wk` by key (keys <= max_key); on success `keys` / `vals` point at the sorted arrays.  Returns 0,
// a CUDA error, or -2 (with the message "<who>: the radix sort asks for ...") when CUB asks for more scratch than the
// workspace reserves.  CUB's kernels are not this library's: they are not counted as its launches.
inline int sort_pairs(const Work& wk, long long L, long long max_key, const char* who, const uint32_t** keys,
                      const uint32_t** vals, cudaStream_t stream) {
  int end_bit = 0;
  while (end_bit < 32 && (max_key >> end_bit) != 0) ++end_bit;
  cub::DoubleBuffer<uint32_t> kb(wk.keys0, wk.keys1), vb(wk.vals0, wk.vals1);
  size_t need = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, need, kb, vb, static_cast<int>(L), 0, end_bit, stream);
  if (e != cudaSuccess) return static_cast<int>(e);
  if (need > wk.temp_bytes) {
    set_error("%s: the radix sort asks for %zu bytes of scratch, the workspace reserves %zu", who, need, wk.temp_bytes);
    return -2;
  }
  e = cub::DeviceRadixSort::SortPairs(wk.temp, need, kb, vb, static_cast<int>(L), 0, end_bit, stream);
  if (e != cudaSuccess) return static_cast<int>(e);
  *keys = kb.Current();
  *vals = vb.Current();
  return 0;
}

}  // namespace scatter
}  // namespace e2f
