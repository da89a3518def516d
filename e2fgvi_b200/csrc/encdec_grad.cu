// Element-wise pieces of the encoder / decoder backward (the convs' input and weight gradients are conv.cu and
// dis_wgrad.cu):
//   upsample2x_backward : adjoint of F.interpolate(scale_factor=2, bilinear, align_corners=True) (the decoder's deconv,
//                         e2fgvi.py:125-129) as a deterministic gather — each input pixel sums the output pixels that
//                         sample it, in a fixed order, no atomics — optionally times LeakyReLU(slope)'s derivative
//   tanh_backward_rows  : dY = dOut * (1 - out^2) of the prediction's tanh (e2fgvi.py:262), written as the row-gapped
//                         operand of the output conv's input gradient and as fp32 NHWC for its weight gradient
//   leaky_backward      : dX = dY * LeakyReLU(slope)'(act), fp32 and its bf16 split
// fp32 arithmetic; the (hi, lo) splits are the operands of the following bf16x3 conv.
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {

namespace {

__device__ __forceinline__ void split8(const float (&f)[8], __nv_bfloat16* hi, __nv_bfloat16* lo) {
  uint32_t hp[4], lp[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 hb = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    const float2 hf = __bfloat1622float2(hb);
    const __nv_bfloat162 lb = __floats2bfloat162_rn(f[2 * i] - hf.x, f[2 * i + 1] - hf.y);
    hp[i] = *reinterpret_cast<const uint32_t*>(&hb);
    lp[i] = *reinterpret_cast<const uint32_t*>(&lb);
  }
  *reinterpret_cast<uint4*>(hi) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
  *reinterpret_cast<uint4*>(lo) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
}

// Weight with which output index o (source coordinate r * o, as the forward computes it) samples input index i of an
// axis of n inputs: (1 - l) at the lower neighbour, l at the upper one, both at the last index.
__device__ __forceinline__ float up_weight(int o, int i, int n, float r) {
  const float s = r * o;
  const int i0 = static_cast<int>(s);
  const int i1 = i0 + ((i0 < n - 1) ? 1 : 0);
  const float l = s - i0;
  return (i0 == i ? 1.f - l : 0.f) + (i1 == i ? l : 0.f);
}

// One thread per (input pixel, 8 channels); grid = (x blocks, input row, image).  Output index o samples inputs
// floor(r o) and floor(r o) + 1 with r = (n - 1) / (2n - 1) < 1/2, so input i is sampled by o in [2i - 2, 2i + 2]; the
// window below is one wider on each side and skips zero weights.
constexpr int UP_R = 3;
__global__ void __launch_bounds__(256) upsample2x_backward_kernel(const float* __restrict__ dy, const float* __restrict__ act,
                                                                  float* __restrict__ dx, __nv_bfloat16* __restrict__ hi,
                                                                  __nv_bfloat16* __restrict__ lo, int H, int W, int C,
                                                                  float rh, float rw, float slope) {
  const int OH = 2 * H, OW = 2 * W, V = C / 8;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= W * V) return;
  const int x = t / V, v = t - x * V;
  const int y = blockIdx.y;
  const long long n = blockIdx.z;
  float wx[2 * UP_R + 1];
#pragma unroll
  for (int j = 0; j <= 2 * UP_R; ++j) {
    const int ox = 2 * x - UP_R + j;
    wx[j] = (ox >= 0 && ox < OW) ? up_weight(ox, x, W, rw) : 0.f;
  }
  float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int jy = 0; jy <= 2 * UP_R; ++jy) {
    const int oy = 2 * y - UP_R + jy;
    if (oy < 0 || oy >= OH) continue;
    const float wy = up_weight(oy, y, H, rh);
    if (wy == 0.f) continue;
#pragma unroll
    for (int jx = 0; jx <= 2 * UP_R; ++jx) {
      if (wx[jx] == 0.f) continue;
      const float wgt = wy * wx[jx];
      const float4* p = reinterpret_cast<const float4*>(dy + ((n * OH + oy) * OW + 2 * x - UP_R + jx) * C + v * 8);
      const float4 a = __ldg(p), b = __ldg(p + 1);
      f[0] += wgt * a.x; f[1] += wgt * a.y; f[2] += wgt * a.z; f[3] += wgt * a.w;
      f[4] += wgt * b.x; f[5] += wgt * b.y; f[6] += wgt * b.z; f[7] += wgt * b.w;
    }
  }
  const long long o = ((n * H + y) * W + x) * C + v * 8;
  if (act) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(act + o)), b = __ldg(reinterpret_cast<const float4*>(act + o) + 1);
    const float av[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (!(av[i] > 0.f)) f[i] *= slope;
  }
  if (dx) {
    reinterpret_cast<float4*>(dx + o)[0] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(dx + o)[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
  if (hi) split8(f, hi + o, lo + o);
}

// One thread per pixel of the row-gapped operand [N][H][pitch][8] + tail (gaps, tail and channels >= C are zero);
// pixels inside the image also write dy32 [N][H][W][8].
__global__ void __launch_bounds__(256) tanh_backward_rows_kernel(const float* __restrict__ dout, const float* __restrict__ out,
                                                                 float* __restrict__ dy32, __nv_bfloat16* __restrict__ hi,
                                                                 __nv_bfloat16* __restrict__ lo, int N, int C, int H, int W,
                                                                 int lead, int pitch, int tail) {
  const long long total = static_cast<long long>(N) * H * pitch + tail;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long row = i / pitch;
  const int xp = static_cast<int>(i - row * pitch) - lead;
  const bool inside = row < static_cast<long long>(N) * H && xp >= 0 && xp < W;
  const long long n = row / H;
  const int y = static_cast<int>(row - n * H);
  float f[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    f[c] = 0.f;
    if (inside && c < C) {
      const long long e = ((n * C + c) * H + y) * static_cast<long long>(W) + xp;
      const float o = __ldg(out + e);
      f[c] = __ldg(dout + e) * (1.f - o * o);
    }
  }
  split8(f, hi + i * 8, lo + i * 8);
  if (inside) {
    float4* d = reinterpret_cast<float4*>(dy32 + (row * W + xp) * 8);
    d[0] = make_float4(f[0], f[1], f[2], f[3]);
    d[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
}

// 8 elements per thread
__global__ void __launch_bounds__(256) leaky_backward_kernel(const float* __restrict__ dy, const float* __restrict__ act,
                                                             float* __restrict__ dx, __nv_bfloat16* __restrict__ hi,
                                                             __nv_bfloat16* __restrict__ lo, long long groups8, float slope) {
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= groups8) return;
  const long long o = g * 8;
  const float4 a0 = __ldg(reinterpret_cast<const float4*>(dy + o)), a1 = __ldg(reinterpret_cast<const float4*>(dy + o) + 1);
  const float4 b0 = __ldg(reinterpret_cast<const float4*>(act + o)), b1 = __ldg(reinterpret_cast<const float4*>(act + o) + 1);
  const float av[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  float f[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (!(av[i] > 0.f)) f[i] *= slope;
  if (dx) {
    reinterpret_cast<float4*>(dx + o)[0] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(dx + o)[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
  if (hi) split8(f, hi + o, lo + o);
}

}  // namespace

int launch_upsample2x_backward(const float* dy, const float* act, float* dx, void* hi, void* lo, int n, int h, int w, int c,
                               float slope, cudaStream_t stream) {
  if (static_cast<long long>(n) * h * w == 0) return 0;
  if (n > 65535 || h > 65535) {
    set_error("upsample2x_backward: at most 65535 images / input rows per launch (got %d, %d)", n, h);
    return -2;
  }
  const int threads = 256, row_threads = w * (c / 8);
  const dim3 grid((row_threads + threads - 1) / threads, h, n);
  // the forward's ratios (launch_upsample2x_split)
  const float rh = (2 * h > 1) ? static_cast<float>(h - 1) / static_cast<float>(2 * h - 1) : 0.f;
  const float rw = (2 * w > 1) ? static_cast<float>(w - 1) / static_cast<float>(2 * w - 1) : 0.f;
  upsample2x_backward_kernel<<<grid, threads, 0, stream>>>(dy, act, dx, static_cast<__nv_bfloat16*>(hi),
                                                           static_cast<__nv_bfloat16*>(lo), h, w, c, rh, rw, slope);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_tanh_backward_rows(const float* dout, const float* out, float* dy32, void* hi, void* lo, int n, int c, int h, int w,
                              int lead, cudaStream_t stream) {
  const int pitch = conv_rows_pitch(w, lead, 8), tail = conv_rows_tail(lead, 8);
  const long long total = static_cast<long long>(n) * h * pitch + tail;
  tanh_backward_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      dout, out, dy32, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), n, c, h, w, lead, pitch, tail);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_leaky_backward(const float* dy, const float* act, float* dx, void* hi, void* lo, long long count, float slope,
                          cudaStream_t stream) {
  const long long g = count / 8;
  if (g == 0) return 0;
  leaky_backward_kernel<<<static_cast<unsigned>((g + 255) / 256), 256, 0, stream>>>(
      dy, act, dx, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), g, slope);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
