// Video-level driver kernels (SURVEY §8(f) rank 4; reference test.py:132-179): everything the reference does on the
// host / in eager torch around each InpaintGenerator.forward call, as byte-exact HBM-bound kernels on uint8 frames.
//
//  * video_prepare_clip : gather the window's frames by id, uint8 -> float / 255 * 2 - 1, multiply by (1 - mask),
//                         mirror-pad to the model's modulus (test.py:139,152-165: to_tensors, imgs * (1 - masks),
//                         cat(x, flip(x))[:h + h_pad] twice) -> masked_frames [t][3][Hp][Wp] fp32 in one pass.
//  * video_compose      : prediction -> ((p + 1) / 2) * 255 -> uint8 (truncation) -> hole composite with the original
//                         frame (test.py:167-174) -> img [n_local][H][W][3] uint8.
//  * video_blend        : comp = first ? img : comp * 0.5 + img * 0.5 in fp32 (test.py:175-179); exact, because every
//                         value is an integer / 2^k with k <= 3.
//  * video_finalize     : fp32 -> uint8 truncation (test.py:195).
// Integer / byte work: results are bit-identical to the reference's numpy code (IEEE fp32 division and rounding
// replicated with __fdiv_rn / separate multiplies, no FMA contraction).
//
// The front end of test.py, run once per video before the window loop:
//  * video_resize_bicubic : PIL Image.resize(size) of uint8 RGB frames with the default BICUBIC filter
//                           (test.py:98-103), Pillow's fixed-point separable resample: horizontal pass into a uint8
//                           intermediate, then the vertical pass; every output byte is
//                           clamp((2^21 + sum_j k_j * in[first + j]) >> 22, 0, 255) in int32.  The (first, count,
//                           k_j) tables come from the host (e2fgvi_b200/video.py).
//  * video_prepare_masks  : read_mask after decoding (test.py:56-70): NEAREST gather through row / column source
//                           tables, > 0, then cv2.dilate with a 3x3 cross 4 times, i.e. 1 iff some in-frame pixel
//                           within L1 distance 4 is set.
#include <cstdint>
#include "launch.h"

namespace e2f {
namespace video {

// one thread per output pixel (x fastest -> coalesced fp32 plane stores); 3 channels per thread
__global__ void __launch_bounds__(256) prepare_clip_kernel(const uint8_t* __restrict__ frames,
                                                           const uint8_t* __restrict__ masks,
                                                           const int* __restrict__ ids, float* __restrict__ out, int t,
                                                           int h, int w, int hp, int wp) {
  const long long total = static_cast<long long>(t) * hp * wp;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = static_cast<int>(i % wp);
  const long long r = i / wp;
  const int y = static_cast<int>(r % hp), k = static_cast<int>(r / hp);
  // cat([x, flip(x)])[:h + pad]: row h + j is row h - 1 - j
  const int sy = y < h ? y : 2 * h - 1 - y, sx = x < w ? x : 2 * w - 1 - x;
  const long long src = (static_cast<long long>(__ldg(ids + k)) * h + sy) * w + sx;
  const float keep = 1.0f - static_cast<float>(__ldg(masks + src) != 0);
  const uint8_t* px = frames + src * 3;
  const long long plane = static_cast<long long>(hp) * wp;
  float* o = out + static_cast<long long>(k) * 3 * plane + static_cast<long long>(y) * wp + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = __fsub_rn(__fmul_rn(__fdiv_rn(static_cast<float>(__ldg(px + c)), 255.0f), 2.0f), 1.0f);
    o[c * plane] = __fmul_rn(v, keep);
  }
}

__global__ void __launch_bounds__(256) compose_kernel(const float* __restrict__ pred, const uint8_t* __restrict__ frames,
                                                      const uint8_t* __restrict__ masks, const int* __restrict__ ids,
                                                      uint8_t* __restrict__ img, int n_local, int h, int w, int hp,
                                                      int wp) {
  const long long total = static_cast<long long>(n_local) * h * w;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = static_cast<int>(i % w);
  const long long r = i / w;
  const int y = static_cast<int>(r % h), k = static_cast<int>(r / h);
  const long long src = (static_cast<long long>(__ldg(ids + k)) * h + y) * w + x;
  const bool hole = __ldg(masks + src) != 0;
  const long long plane = static_cast<long long>(hp) * wp;
  const float* p = pred + static_cast<long long>(k) * 3 * plane + static_cast<long long>(y) * wp + x;
  uint8_t* o = img + i * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    uint8_t v;
    if (hole) {
      const float f = __fmul_rn(__fdiv_rn(__fadd_rn(__ldg(p + c * plane), 1.0f), 2.0f), 255.0f);
      v = static_cast<uint8_t>(static_cast<int>(f));          // numpy astype(uint8): truncation; f is in [0, 255]
    } else {
      v = __ldg(frames + src * 3 + c);
    }
    o[c] = v;
  }
}

// one thread per byte of img
__global__ void __launch_bounds__(256) blend_kernel(const uint8_t* __restrict__ img, const int* __restrict__ ids,
                                                    const int* __restrict__ first, float* __restrict__ comp,
                                                    int n_local, long long frame_elems) {
  const long long total = static_cast<long long>(n_local) * frame_elems;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = static_cast<int>(i / frame_elems);
  const long long e = i - static_cast<long long>(k) * frame_elems;
  float* c = comp + static_cast<long long>(__ldg(ids + k)) * frame_elems + e;
  const float v = static_cast<float>(__ldg(img + i));
  *c = __ldg(first + k) ? v : __fadd_rn(__fmul_rn(*c, 0.5f), __fmul_rn(v, 0.5f));
}

__global__ void __launch_bounds__(256) finalize_kernel(const float* __restrict__ comp, uint8_t* __restrict__ out,
                                                       long long count) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < count) out[i] = static_cast<uint8_t>(static_cast<int>(__ldg(comp + i)));
}

static unsigned blocks_for(long long total) { return static_cast<unsigned>((total + 255) / 256); }

// ------------------------------------------------------------------------------------------------ bicubic resize
// Pillow's 8-bit resample (libImaging/Resample.c): 22 fractional bits, int32 sums started at half an output step.
constexpr int kResamplePrecision = 22;

__device__ __forceinline__ uint8_t clip8(int acc) {
  const int v = acc >> kResamplePrecision;                     // arithmetic shift, like Pillow's clip8
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Horizontal pass, one block per image row: the row (w * 3 bytes) is staged in shared memory with 16-byte loads when
// the row is 16-byte aligned, so every input byte is read from HBM once; each thread then produces whole RGB output
// pixels from the table row [first, count, k_0 .. k_{taps-1}] of its output column.
__global__ void __launch_bounds__(256) resize_h_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                       const int* __restrict__ xtab, int taps, int w, int w2) {
  extern __shared__ __align__(16) uint8_t row[];
  const long long r = blockIdx.x;
  const int in_bytes = w * 3, out_bytes = w2 * 3;
  const uint8_t* s = src + r * in_bytes;
  if ((reinterpret_cast<uintptr_t>(s) & 15) == 0) {
    const int n16 = in_bytes >> 4;
    for (int i = threadIdx.x; i < n16; i += blockDim.x)
      reinterpret_cast<uint4*>(row)[i] = __ldg(reinterpret_cast<const uint4*>(s) + i);
    for (int i = (n16 << 4) + threadIdx.x; i < in_bytes; i += blockDim.x) row[i] = __ldg(s + i);
  } else {
    for (int i = threadIdx.x; i < in_bytes; i += blockDim.x) row[i] = __ldg(s + i);
  }
  __syncthreads();
  uint8_t* d = dst + r * out_bytes;
  const int stride = taps + 2;
  for (int x = threadIdx.x; x < w2; x += blockDim.x) {
    const int* t = xtab + static_cast<long long>(x) * stride;
    const int first = __ldg(t), count = min(__ldg(t + 1), taps);
    int a0 = 1 << (kResamplePrecision - 1), a1 = a0, a2 = a0;
    const uint8_t* p = row + first * 3;
    for (int j = 0; j < count; ++j) {
      const int k = __ldg(t + 2 + j);
      a0 += static_cast<int>(p[3 * j]) * k;
      a1 += static_cast<int>(p[3 * j + 1]) * k;
      a2 += static_cast<int>(p[3 * j + 2]) * k;
    }
    d[3 * x] = clip8(a0);
    d[3 * x + 1] = clip8(a1);
    d[3 * x + 2] = clip8(a2);
  }
}

// Vertical pass: blockIdx.x = output row (image-major), threads along the row's bytes (coalesced); the taps of a row
// are consecutive source rows, mostly L2-resident because neighbouring output rows share them.
__global__ void __launch_bounds__(256) resize_v_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                       const int* __restrict__ ytab, int taps, int h, int h2,
                                                       int row_bytes) {
  const int e = blockIdx.y * blockDim.x + threadIdx.x;
  if (e >= row_bytes) return;
  const long long r = blockIdx.x;
  const long long img = r / h2;
  const int y = static_cast<int>(r - img * h2);
  const int* t = ytab + static_cast<long long>(y) * (taps + 2);
  const int first = __ldg(t), count = min(__ldg(t + 1), taps);
  const uint8_t* s = src + (img * h + first) * row_bytes + e;
  int acc = 1 << (kResamplePrecision - 1);
  for (int j = 0; j < count; ++j) acc += static_cast<int>(__ldg(s + static_cast<long long>(j) * row_bytes)) * __ldg(t + 2 + j);
  dst[r * row_bytes + e] = clip8(acc);
}

// ------------------------------------------------------------------------------------------------ mask preparation
constexpr int kMaskTile = 32, kMaskHalo = 4, kMaskSpan = kMaskTile + 2 * kMaskHalo;

// One block per 32 x 32 output tile (loops over images along z): the tile plus a 4-pixel halo is gathered through the
// NEAREST tables and binarised into shared memory (outside the frame = 0), then every output pixel ORs the 41 pixels
// of its L1 ball of radius 4 (= four 3x3-cross dilations, which never need out-of-frame pixels: a monotone path
// between two in-frame pixels stays inside the frame).
__global__ void __launch_bounds__(256) prepare_masks_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                            const int* __restrict__ rows, const int* __restrict__ cols,
                                                            int n, int hm, int wm, int h, int w) {
  __shared__ uint8_t tile[kMaskSpan][kMaskSpan];
  const int x0 = blockIdx.x * kMaskTile, y0 = blockIdx.y * kMaskTile;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthreads = blockDim.x * blockDim.y;
  for (int img = blockIdx.z; img < n; img += gridDim.z) {
    const uint8_t* s = src + static_cast<long long>(img) * hm * wm;
    for (int i = tid; i < kMaskSpan * kMaskSpan; i += nthreads) {
      const int ty = i / kMaskSpan, tx = i - ty * kMaskSpan;
      const int y = y0 - kMaskHalo + ty, x = x0 - kMaskHalo + tx;
      uint8_t v = 0;
      if (y >= 0 && y < h && x >= 0 && x < w)
        v = __ldg(s + static_cast<long long>(__ldg(rows + y)) * wm + __ldg(cols + x)) != 0;
      tile[ty][tx] = v;
    }
    __syncthreads();
    uint8_t* d = dst + static_cast<long long>(img) * h * w;
    const int tx = threadIdx.x;
    for (int ty = threadIdx.y; ty < kMaskTile; ty += blockDim.y) {
      const int y = y0 + ty, x = x0 + tx;
      uint8_t v = 0;
#pragma unroll
      for (int dy = -kMaskHalo; dy <= kMaskHalo; ++dy) {
        const int r = kMaskHalo - (dy < 0 ? -dy : dy);
#pragma unroll
        for (int dx = -r; dx <= r; ++dx) v |= tile[ty + kMaskHalo + dy][tx + kMaskHalo + dx];
      }
      if (y < h && x < w) d[static_cast<long long>(y) * w + x] = v;
    }
    __syncthreads();
  }
}

}  // namespace video

int launch_video_prepare_clip(const uint8_t* frames, const uint8_t* masks, const int* ids, float* out, int t, int h,
                              int w, int hp, int wp, cudaStream_t stream) {
  const long long total = static_cast<long long>(t) * hp * wp;
  if (total == 0) return 0;
  video::prepare_clip_kernel<<<video::blocks_for(total), 256, 0, stream>>>(frames, masks, ids, out, t, h, w, hp, wp);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_video_compose(const float* pred, const uint8_t* frames, const uint8_t* masks, const int* ids, uint8_t* img,
                         int n_local, int h, int w, int hp, int wp, cudaStream_t stream) {
  const long long total = static_cast<long long>(n_local) * h * w;
  if (total == 0) return 0;
  video::compose_kernel<<<video::blocks_for(total), 256, 0, stream>>>(pred, frames, masks, ids, img, n_local, h, w, hp, wp);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_video_blend(const uint8_t* img, const int* ids, const int* first, float* comp, int n_local,
                       long long frame_elems, cudaStream_t stream) {
  const long long total = static_cast<long long>(n_local) * frame_elems;
  if (total == 0) return 0;
  video::blend_kernel<<<video::blocks_for(total), 256, 0, stream>>>(img, ids, first, comp, n_local, frame_elems);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_video_finalize(const float* comp, uint8_t* out, long long count, cudaStream_t stream) {
  if (count == 0) return 0;
  video::finalize_kernel<<<video::blocks_for(count), 256, 0, stream>>>(comp, out, count);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_video_resize_bicubic(const uint8_t* src, uint8_t* dst, uint8_t* scratch, const int* xtab, int xtaps,
                                const int* ytab, int ytaps, int n, int h, int w, int h2, int w2, cudaStream_t stream) {
  if (n == 0) return 0;
  const bool horiz = w2 != w, vert = h2 != h;
  if (!horiz && !vert)
    return static_cast<int>(cudaMemcpyAsync(dst, src, static_cast<size_t>(n) * h * w * 3, cudaMemcpyDeviceToDevice, stream));
  if (horiz) {
    const int smem = (w * 3 + 15) & ~15;
    if (smem > 48 * 1024) {
      const cudaError_t e = cudaFuncSetAttribute(video::resize_h_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      if (e != cudaSuccess) return static_cast<int>(e);
    }
    video::resize_h_kernel<<<static_cast<unsigned>(static_cast<long long>(n) * h), 256, smem, stream>>>(
        src, vert ? scratch : dst, xtab, xtaps, w, w2);
    count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (vert) {
    const int row_bytes = w2 * 3;
    const dim3 grid(static_cast<unsigned>(static_cast<long long>(n) * h2), static_cast<unsigned>((row_bytes + 255) / 256));
    video::resize_v_kernel<<<grid, 256, 0, stream>>>(horiz ? scratch : src, dst, ytab, ytaps, h, h2, row_bytes);
    count_launch();
  }
  return static_cast<int>(cudaGetLastError());
}

int launch_video_prepare_masks(const uint8_t* src, uint8_t* dst, const int* rows, const int* cols, int n, int hm,
                               int wm, int h, int w, cudaStream_t stream) {
  if (n == 0) return 0;
  const dim3 grid(static_cast<unsigned>((w + video::kMaskTile - 1) / video::kMaskTile),
                  static_cast<unsigned>((h + video::kMaskTile - 1) / video::kMaskTile),
                  static_cast<unsigned>(n < 65535 ? n : 65535));
  video::prepare_masks_kernel<<<grid, dim3(video::kMaskTile, 8), 0, stream>>>(src, dst, rows, cols, n, hm, wm, h, w);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
