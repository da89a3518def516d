// flow_warp: bilinear gather at (x + u, y + v)  — reference model/modules/flow_comp.py:345-383.
// HBM-bound: per output pixel 4 corner reads of C channels + one write.  NHWC layout makes every corner read a
// contiguous C*sizeof(T) run, so a warp reads whole 128B lines with 16-byte vectors.
// Algorithmic bytes per call (SURVEY §8d): (2*C + 2) * H*W * 4  (fp32), i.e. x read once + out written once + flow.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "flow_warp_math.cuh"
#include "launch.h"

namespace e2f {

// One thread per (pixel, 16-byte channel vector).
template <typename T>
__global__ void __launch_bounds__(256) flow_warp_nhwc_kernel(const T* __restrict__ x, const float2* __restrict__ flow,
                                                             T* __restrict__ out, int N, int H, int W, int C,
                                                             int pad_mode) {
  constexpr int VEC = 16 / sizeof(T);
  const int vecs = C / VEC;
  const long long total = static_cast<long long>(N) * H * W * vecs;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int v = static_cast<int>(idx % vecs);
  const long long pix = idx / vecs;
  const int xw = static_cast<int>(pix % W);
  const int yh = static_cast<int>((pix / W) % H);
  const long long n = pix / (static_cast<long long>(W) * H);
  const float2 f = __ldg(flow + pix);
  const Corner c = make_corners(static_cast<float>(xw) + f.x, static_cast<float>(yh) + f.y, H, W, pad_mode);
  const T* base = x + n * H * W * C + v * VEC;
  uint4 raw[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) raw[k] = __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(c.off[k]) * C));
  uint4 res;
  if constexpr (sizeof(T) == 4) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float* p = reinterpret_cast<const float*>(&raw[k]);
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = fmaf(c.wgt[k], p[i], acc[i]);
    }
    res = *reinterpret_cast<uint4*>(acc);
  } else {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __half2* p = reinterpret_cast<const __half2*>(&raw[k]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(p[i]);
        acc[2 * i] = fmaf(c.wgt[k], t.x, acc[2 * i]);
        acc[2 * i + 1] = fmaf(c.wgt[k], t.y, acc[2 * i + 1]);
      }
    }
    uint32_t* r = reinterpret_cast<uint32_t*>(&res);
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = pack_half2(acc[2 * i], acc[2 * i + 1]);
  }
  *reinterpret_cast<uint4*>(out + pix * C + v * VEC) = res;
}

// NCHW fp32, any (small) C: one thread per pixel, channel loop.  Used for 2-channel flows and 3-channel images.
__global__ void __launch_bounds__(256) flow_warp_nchw_kernel(const float* __restrict__ x, const float2* __restrict__ flow,
                                                             float* __restrict__ out, int N, int C, int H, int W,
                                                             int pad_mode) {
  const long long total = static_cast<long long>(N) * H * W;
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const int xw = static_cast<int>(pix % W);
  const int yh = static_cast<int>((pix / W) % H);
  const long long n = pix / (static_cast<long long>(W) * H);
  const float2 f = __ldg(flow + pix);
  const Corner c = make_corners(static_cast<float>(xw) + f.x, static_cast<float>(yh) + f.y, H, W, pad_mode);
  const long long plane = static_cast<long long>(H) * W;
  const float* xb = x + n * C * plane;
  float* ob = out + n * C * plane + static_cast<long long>(yh) * W + xw;
  for (int ch = 0; ch < C; ++ch) {
    const float* p = xb + ch * plane;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) acc = fmaf(c.wgt[k], __ldg(p + c.off[k]), acc);
    ob[ch * plane] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused prologue of one propagation step (SURVEY 8(f) rank 3; reference feat_prop.py:106-126): everything the step
// does before its offset-head conv and its DCN, in ONE pass over the two feature maps:
//   cond_n1 = flow_warp(feat_prop, flow_n1)                               -> bf16 (hi, lo) split, conv operand
//   flow_n2 = flow_n1 + flow_warp(flows[:, i-2], flow_n1)                 -> fp32 [N][H][W][2] (DCN operand)
//   cond_n2 = flow_warp(feat_n2, flow_n2)                                 -> bf16 (hi, lo) split
//   cat([flow_n1, flow_n2], 1)                                            -> 8-channel (4 + zero pad) bf16 split, conv operand
//   cat([feat_prop, feat_n2], 1)                                          -> fp16 group-major [N][2C/16][H][W][16], DCN input
// replacing 3 flow_warp launches, an add, 3 layout copies, a cat, 3 split launches, the pack launch and (first step)
// three zero fills.  The arithmetic of every output is the arithmetic of the kernels it replaces (same fmaf order in the
// bilinear blend, same rounding in the splits), so the results are bit-identical to the unfused path.
// One thread per (pixel, 4-channel vector); feat_n2 / flow_prev may be null (second frame of a sweep: zeros).
__global__ void __launch_bounds__(256)
prop_prologue_kernel(const float* __restrict__ prop, const float* __restrict__ feat2, const float* __restrict__ flow1,
                     long long f1_bs, const float* __restrict__ flowp, long long fp_bs, __nv_bfloat16* __restrict__ c1h,
                     __nv_bfloat16* __restrict__ c1l, __nv_bfloat16* __restrict__ c2h, __nv_bfloat16* __restrict__ c2l,
                     float2* __restrict__ f1_out, float2* __restrict__ f2_out, __nv_bfloat16* __restrict__ flh,
                     __nv_bfloat16* __restrict__ fll, __half* __restrict__ xg, int N, int H, int W, int C) {
  const int vecs = C / 4;
  const long long total = static_cast<long long>(N) * H * W * vecs;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int v = static_cast<int>(idx % vecs);
  const long long pix = idx / vecs;
  const int xw = static_cast<int>(pix % W);
  const int yh = static_cast<int>((pix / W) % H);
  const long long n = pix / (static_cast<long long>(W) * H);
  const long long plane = static_cast<long long>(H) * W;
  const long long pl = static_cast<long long>(yh) * W + xw;
  const float u1 = __ldg(flow1 + n * f1_bs + pl), v1 = __ldg(flow1 + n * f1_bs + plane + pl);
  const Corner c = make_corners(static_cast<float>(xw) + u1, static_cast<float>(yh) + v1, H, W, 0);

  auto gather = [&](const float* src, const Corner& cc, float (&acc)[4]) {
    const float* base = src + n * plane * C + v * 4;
    uint4 raw[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) raw[k] = __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(cc.off[k]) * C));
    acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float* p = reinterpret_cast<const float*>(&raw[k]);
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = fmaf(cc.wgt[k], p[i], acc[i]);
    }
  };
  auto store_split4 = [&](const float (&a)[4], __nv_bfloat16* hi, __nv_bfloat16* lo, long long elem) {
    __align__(8) __nv_bfloat16 h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      h[e] = __float2bfloat16_rn(a[e]);
      l[e] = __float2bfloat16_rn(a[e] - __bfloat162float(h[e]));
    }
    *reinterpret_cast<uint2*>(hi + elem) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(lo + elem) = *reinterpret_cast<const uint2*>(l);
  };

  float acc[4];
  gather(prop, c, acc);
  store_split4(acc, c1h, c1l, pix * C + v * 4);

  float u2 = 0.f, v2 = 0.f;
  if (feat2 != nullptr) {
    const float* pb = flowp + n * fp_bs;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      a0 = fmaf(c.wgt[k], __ldg(pb + c.off[k]), a0);
      a1 = fmaf(c.wgt[k], __ldg(pb + plane + c.off[k]), a1);
    }
    u2 = u1 + a0;
    v2 = v1 + a1;
    const Corner c2 = make_corners(static_cast<float>(xw) + u2, static_cast<float>(yh) + v2, H, W, 0);
    gather(feat2, c2, acc);
  } else {
    acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
  }
  store_split4(acc, c2h, c2l, pix * C + v * 4);

  // DCN input: this pixel's own (unwarped) values, fp16, group-major (16 channels = 4 vectors per group)
  const int G = 2 * C / 16;
  {
    const float4 pc = __ldg(reinterpret_cast<const float4*>(prop + pix * C + v * 4));
    const uint2 o = make_uint2(pack_half2(pc.x, pc.y), pack_half2(pc.z, pc.w));
    *reinterpret_cast<uint2*>(xg + ((n * G + v / 4) * plane + pl) * 16 + (v % 4) * 4) = o;
    uint2 o2 = make_uint2(0u, 0u);
    if (feat2 != nullptr) {
      const float4 fc = __ldg(reinterpret_cast<const float4*>(feat2 + pix * C + v * 4));
      o2 = make_uint2(pack_half2(fc.x, fc.y), pack_half2(fc.z, fc.w));
    }
    *reinterpret_cast<uint2*>(xg + ((n * G + C / 16 + v / 4) * plane + pl) * 16 + (v % 4) * 4) = o2;
  }
  if (v == 0) {
    f1_out[pix] = make_float2(u1, v1);
    f2_out[pix] = make_float2(u2, v2);
    const float fl[4] = {u1, v1, u2, v2};
    store_split4(fl, flh, fll, pix * 8);
    const uint2 z = make_uint2(0u, 0u);
    *reinterpret_cast<uint2*>(flh + pix * 8 + 4) = z;
    *reinterpret_cast<uint2*>(fll + pix * 8 + 4) = z;
  }
}

int launch_flow_warp_nhwc(const void* x, const float* flow, void* out, int n, int h, int w, int c, int dtype,
                          int pad_mode, cudaStream_t stream) {
  const int vec = dtype == 1 ? 8 : 4;
  const long long total = static_cast<long long>(n) * h * w * (c / vec);
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
  if (blocks == 0) return 0;
  if (dtype == 1)
    flow_warp_nhwc_kernel<__half><<<blocks, threads, 0, stream>>>(static_cast<const __half*>(x),
                                                                   reinterpret_cast<const float2*>(flow),
                                                                   static_cast<__half*>(out), n, h, w, c, pad_mode);
  else
    flow_warp_nhwc_kernel<float><<<blocks, threads, 0, stream>>>(static_cast<const float*>(x),
                                                                  reinterpret_cast<const float2*>(flow),
                                                                  static_cast<float*>(out), n, h, w, c, pad_mode);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_flow_warp_nchw(const float* x, const float* flow, float* out, int n, int c, int h, int w, int pad_mode,
                          cudaStream_t stream) {
  const long long total = static_cast<long long>(n) * h * w;
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
  if (blocks == 0) return 0;
  flow_warp_nchw_kernel<<<blocks, threads, 0, stream>>>(x, reinterpret_cast<const float2*>(flow), out, n, c, h, w,
                                                        pad_mode);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_prop_prologue(const float* prop, const float* feat2, const float* flow1, long long f1_bs, const float* flowp,
                         long long fp_bs, void* c1h, void* c1l, void* c2h, void* c2l, float* f1_out, float* f2_out,
                         void* flh, void* fll, void* xg, int n, int h, int w, int c, cudaStream_t stream) {
  const long long total = static_cast<long long>(n) * h * w * (c / 4);
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
  if (blocks == 0) return 0;
  prop_prologue_kernel<<<blocks, threads, 0, stream>>>(
      prop, feat2, flow1, f1_bs, flowp, fp_bs, static_cast<__nv_bfloat16*>(c1h), static_cast<__nv_bfloat16*>(c1l),
      static_cast<__nv_bfloat16*>(c2h), static_cast<__nv_bfloat16*>(c2l), reinterpret_cast<float2*>(f1_out),
      reinterpret_cast<float2*>(f2_out), static_cast<__nv_bfloat16*>(flh), static_cast<__nv_bfloat16*>(fll),
      static_cast<__half*>(xg), n, h, w, c);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
