// The deformable sampler's offset / mask activations, shared by the forward (dcn.cu) and its adjoint (dcn_grad.cu):
// the backward recomputes offsets and masks with the very instructions the forward used.
#pragma once
#include <cuda_runtime.h>

namespace e2f {
namespace dcn {

__device__ __forceinline__ float fast_tanh(float v) {
  // 1 - 2/(e^{2v}+1): abs error ~1e-7, saturates cleanly for |v| large
  const float e = __expf(2.f * v);
  return 1.f - __fdividef(2.f, e + 1.f);
}
__device__ __forceinline__ float fast_sigmoid(float v) { return __fdividef(1.f, 1.f + __expf(-v)); }

}  // namespace dcn
}  // namespace e2f
