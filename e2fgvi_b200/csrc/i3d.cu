// I3D (InceptionI3d, the network behind evaluate.py's VFID; reference core/metrics.py:196-570) on sm_90a.
//
//  * The Unit3D convs (conv + eval BatchNorm folded on the host + ReLU) run on conv.cu's implicit-GEMM kernel, its T3
//    instantiation: NDHWC bf16 (hi, lo) operands through 5-D tensor maps, 3-term split, fp32 accumulation; the epilogue
//    writes fp32 and/or the split into a channel slice of a wider output, so an Inception module's torch.cat is never
//    a copy.
//  * The 3-channel 7x7x7 / stride-2 stem runs window-packed: each K chunk is 16 consecutive pixels x 4 channels of one
//    input row (7 taps used), i.e. 49 chunks of 64 instead of 343 taps padded from 3 to 64 channels.  stem_pack_kernel
//    writes that row-gapped operand straight from the uint8 frames (u / 255 in fp32, ToTorchFormatTensor's
//    img.float().div(255)) or from the reference's fp32 (B, 3, T, H, W) input.
//  * MaxPool3dSamePadding: the reference pads with zeros (F.pad) before nn.MaxPool3d, so padded positions take part in
//    the max as 0.  A max of fp32 values: bit-exact.
//  * extract_features' x.mean(4).mean(3).mean(2): one thread per (video, channel), the three means in that order.
#include <cuda_bf16.h>
#include <cstdint>
#include "launch.h"

namespace e2f {
namespace i3d {

__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 g = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - g.x, b - g.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// one thread per pixel of the row-gapped layout [b*t*h][pitch][4] + tail (gaps, tail and channel 3 are zero)
template <bool U8>
__global__ void __launch_bounds__(256) stem_pack_kernel(const void* __restrict__ src, __nv_bfloat16* __restrict__ hi,
                                                        __nv_bfloat16* __restrict__ lo, int b, int t, int h, int w,
                                                        int lead, int pitch, int tail) {
  const long long rows = static_cast<long long>(b) * t * h;
  const long long total = rows * pitch + tail;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long row = i / pitch;
  const int x = static_cast<int>(i - row * pitch) - lead;
  float f[3] = {0.f, 0.f, 0.f};
  if (row < rows && x >= 0 && x < w) {
    if (U8) {
      const uint8_t* px = static_cast<const uint8_t*>(src) + (row * w + x) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) f[c] = static_cast<float>(px[c]) / 255.0f;
    } else {
      const long long y = row % h, bt = row / h, tt = bt % t, bb = bt / t;
      const float* xs = static_cast<const float*>(src);
#pragma unroll
      for (int c = 0; c < 3; ++c) f[c] = __ldg(xs + (((bb * 3 + c) * t + tt) * h + y) * w + x);
    }
  }
  uint32_t h0, l0, h1, l1;
  split2(f[0], f[1], h0, l0);
  split2(f[2], 0.f, h1, l1);
  *reinterpret_cast<uint2*>(hi + i * 4) = make_uint2(h0, h1);
  *reinterpret_cast<uint2*>(lo + i * 4) = make_uint2(l0, l1);
}

struct PoolGeom {
  int b, t, h, w, c;          // input [b][t][h][w][c]
  int to, ho, wo;             // output [b][to][ho][wo][c]
  int kt, kh, kw, st, sh, sw, pt, ph, pw;
};

// one thread per (output pixel, 4 channels)
__global__ void __launch_bounds__(256) maxpool_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                      __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo,
                                                      const PoolGeom g) {
  const int c4 = g.c / 4;
  const long long total = static_cast<long long>(g.b) * g.to * g.ho * g.wo * c4;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int cq = static_cast<int>(i % c4);
  long long r = i / c4;
  const int xo = static_cast<int>(r % g.wo);
  r /= g.wo;
  const int yo = static_cast<int>(r % g.ho);
  r /= g.ho;
  const int to = static_cast<int>(r % g.to);
  const long long bb = r / g.to;
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  bool pad = false;
  for (int kt = 0; kt < g.kt; ++kt) {
    const int ti = to * g.st - g.pt + kt;
    for (int ky = 0; ky < g.kh; ++ky) {
      const int yi = yo * g.sh - g.ph + ky;
      for (int kx = 0; kx < g.kw; ++kx) {
        const int xi = xo * g.sw - g.pw + kx;
        if (ti < 0 || ti >= g.t || yi < 0 || yi >= g.h || xi < 0 || xi >= g.w) {
          pad = true;
          continue;
        }
        const float4 v = __ldg(reinterpret_cast<const float4*>(
                                   x + (((bb * g.t + ti) * g.h + yi) * static_cast<long long>(g.w) + xi) * g.c) + cq);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
  }
  if (pad) {                                  // the zeros F.pad put there
    m.x = fmaxf(m.x, 0.f); m.y = fmaxf(m.y, 0.f); m.z = fmaxf(m.z, 0.f); m.w = fmaxf(m.w, 0.f);
  }
  const long long o = r * static_cast<long long>(g.ho) * g.wo;  // (b, to) image index * pixels
  const long long off = ((o + static_cast<long long>(yo) * g.wo + xo) * g.c) + cq * 4;
  if (out) *reinterpret_cast<float4*>(out + off) = m;
  if (out_hi) {
    uint32_t h0, l0, h1, l1;
    split2(m.x, m.y, h0, l0);
    split2(m.z, m.w, h1, l1);
    *reinterpret_cast<uint2*>(out_hi + off) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(out_lo + off) = make_uint2(l0, l1);
  }
}

// x.mean(4).mean(3).mean(2) of an NDHWC tensor: one thread per (video, channel), fixed summation order
__global__ void __launch_bounds__(256) mean_thw_kernel(const float* __restrict__ x, float* __restrict__ out, int b, int t,
                                                       int h, int w, int c) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(b) * c) return;
  const int ch = static_cast<int>(i % c);
  const long long bb = i / c;
  const float* p = x + bb * t * h * static_cast<long long>(w) * c + ch;
  float st = 0.f;
  for (int tt = 0; tt < t; ++tt) {
    float sh = 0.f;
    for (int y = 0; y < h; ++y) {
      float sw = 0.f;
      for (int xx = 0; xx < w; ++xx, p += c) sw += __ldg(p);
      sh += sw / w;
    }
    st += sh / h;
  }
  out[i] = st / t;
}

}  // namespace i3d

// compute_pad(k = 7, stride = 2, s): max(7 - 2, 0) when s % 2 == 0, else max(7 - 1, 0); front = pad / 2
static void stem_pad(int s, int* pad_f, int* pad_b) {
  const int pad = s % 2 == 0 ? 5 : 6;
  *pad_f = pad / 2;
  *pad_b = pad - *pad_f;
}

// row-gapped stem operand: lead >= both x paddings with lead - pad_f even (window starts on 16-byte boundaries)
static void i3d_stem_layout(int w, int* lead, int* pitch) {
  int pf, pb;
  stem_pad(w, &pf, &pb);
  int l = pb > pf ? pb : pf;
  if ((l - pf) & 1) ++l;
  *lead = l;
  *pitch = conv_rows_pitch(w, l, 4);
}

long long i3d_stem_elems(int b, int t, int h, int w) {
  int lead, pitch;
  i3d_stem_layout(w, &lead, &pitch);
  return (static_cast<long long>(b) * t * h * pitch + I3D_STEM_TAIL) * 4;
}

int launch_i3d_stem_pack(const void* x, int x_u8, void* hi, void* lo, int b, int t, int h, int w, cudaStream_t stream) {
  int lead, pitch;
  i3d_stem_layout(w, &lead, &pitch);
  const long long total = static_cast<long long>(b) * t * h * pitch + I3D_STEM_TAIL;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  auto* h16 = static_cast<__nv_bfloat16*>(hi);
  auto* l16 = static_cast<__nv_bfloat16*>(lo);
  if (x_u8)
    i3d::stem_pack_kernel<true><<<blocks, 256, 0, stream>>>(x, h16, l16, b, t, h, w, lead, pitch, I3D_STEM_TAIL);
  else
    i3d::stem_pack_kernel<false><<<blocks, 256, 0, stream>>>(x, h16, l16, b, t, h, w, lead, pitch, I3D_STEM_TAIL);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_i3d_stem_conv(const void* hi, const void* lo, const void* w_hi, const void* w_lo, const float* bias, float* out,
                         void* out_hi, void* out_lo, int out_cs, int b, int t, int h, int w, int cout, cudaStream_t stream) {
  int lead, pitch, pad[6];
  i3d_stem_layout(w, &lead, &pitch);
  stem_pad(t, &pad[0], &pad[1]);
  stem_pad(h, &pad[2], &pad[3]);
  stem_pad(w, &pad[4], &pad[5]);
  return launch_conv3d(hi, lo, 4, lead, w_hi, w_lo, bias, out, out_hi, out_lo, out_cs, b, t, h, w, cout, 7, 2, pad, 0.f,
                       stream);
}

int launch_i3d_maxpool(const float* x, float* out, void* out_hi, void* out_lo, int b, int t, int h, int w, int c,
                       const int* k, const int* s, const int* pad, cudaStream_t stream) {
  i3d::PoolGeom g;
  g.b = b; g.t = t; g.h = h; g.w = w; g.c = c;
  g.kt = k[0]; g.kh = k[1]; g.kw = k[2];
  g.st = s[0]; g.sh = s[1]; g.sw = s[2];
  g.pt = pad[0]; g.ph = pad[2]; g.pw = pad[4];
  g.to = (t + pad[0] + pad[1] - k[0]) / s[0] + 1;
  g.ho = (h + pad[2] + pad[3] - k[1]) / s[1] + 1;
  g.wo = (w + pad[4] + pad[5] - k[2]) / s[2] + 1;
  const long long total = static_cast<long long>(b) * g.to * g.ho * g.wo * (c / 4);
  if (total == 0) return 0;
  i3d::maxpool_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      x, out, static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), g);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_i3d_mean(const float* x, float* out, int b, int t, int h, int w, int c, cudaStream_t stream) {
  const long long total = static_cast<long long>(b) * c;
  if (total == 0) return 0;
  i3d::mean_thw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(x, out, b, t, h, w, c);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
