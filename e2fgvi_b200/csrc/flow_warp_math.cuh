// The bilinear corners of flow_warp (zeros / border padding), shared by the warps and the propagation prologue
// (flow_warp.cu) and their adjoint (flow_warp_grad.cu): the backward recomputes the forward's corners and weights with
// the very same instructions.
#pragma once
#include <cuda_runtime.h>

namespace e2f {

struct Corner {
  int off[4];     // pixel offsets (in pixels) of the 4 corners, clamped to be addressable
  float wgt[4];   // bilinear weight, 0 for corners outside the image (zeros padding)
  float lx, ly;   // fractional position inside the cell (the slopes' weights)
  unsigned in;    // bit k: corner k lies inside the image
};

// (px, py): absolute sample position.  pad_mode 0 = zeros, 1 = border (clamp the coordinate first).
__device__ __forceinline__ Corner make_corners(float px, float py, int H, int W, int pad_mode) {
  if (pad_mode == 1) {
    px = fminf(fmaxf(px, 0.f), static_cast<float>(W - 1));
    py = fminf(fmaxf(py, 0.f), static_cast<float>(H - 1));
  }
  // keep the float->int conversion defined for wild flows
  px = fminf(fmaxf(px, -4.f), static_cast<float>(W) + 4.f);
  py = fminf(fmaxf(py, -4.f), static_cast<float>(H) + 4.f);
  const float fx = floorf(px), fy = floorf(py);
  const float lx = px - fx, ly = py - fy;
  const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
  Corner c;
  c.lx = lx;
  c.ly = ly;
  c.in = 0u;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int dy = k >> 1, dx = k & 1;
    const int yy = y0 + dy, xx = x0 + dx;
    const bool in = (yy >= 0) && (yy < H) && (xx >= 0) && (xx < W);
    const float w = (dy ? ly : 1.f - ly) * (dx ? lx : 1.f - lx);
    c.wgt[k] = in ? w : 0.f;
    c.off[k] = min(max(yy, 0), H - 1) * W + min(max(xx, 0), W - 1);
    c.in |= in ? (1u << k) : 0u;
  }
  return c;
}

}  // namespace e2f
