// Backward of flow_warp (flow_warp.cu; zeros padding, align_corners=True, pixel units): given dout, the gradient of
// out = sum_k w_k x[corner_k] at (x + u, y + v),
//   d flow: per pixel sum_c dout[c] (d out[c] / d u, d out[c] / d v), with the floor-based slopes of the bilinear form
//     (a corner outside the image contributes neither value nor slope), summed over the channels in a fixed order: each
//     lane its channels in order, then a shuffle tree over the warp (NHWC), or one thread's channel loop (NCHW);
//   dx: the scatter of w_k dout to the 4 corners, deterministic: the sample kernel writes one (destination pixel, source
//     index (pixel*4 + corner)) pair and the weight per corner (destination M = N*H*W for corners outside the image),
//     CUB's stable radix sort orders the pairs by destination (scatter_sort.cuh), and the gather kernel adds every
//     destination's run in source order, after an optional residual.  No float atomics: a second run gives the same bits.
// The corners come from the forward's make_corners (flow_warp_math.cuh), so they are the forward's to the bit.
#include <cuda_runtime.h>
#include <climits>
#include "common.cuh"
#include "flow_warp_math.cuh"
#include "launch.h"
#include "scatter_sort.cuh"

namespace e2f {
namespace flow_warp_grad {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

__device__ __forceinline__ void write_list(const Corner& c, long long pix, long long img, uint32_t sentinel,
                                           uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                           float* __restrict__ coef) {
  uint32_t kk[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) kk[k] = (c.in >> k & 1u) ? static_cast<uint32_t>(img + c.off[k]) : sentinel;
  const long long idx = pix * 4;
  const uint32_t i0 = static_cast<uint32_t>(idx);
  *reinterpret_cast<uint4*>(keys + idx) = make_uint4(kk[0], kk[1], kk[2], kk[3]);
  *reinterpret_cast<uint4*>(vals + idx) = make_uint4(i0, i0 + 1, i0 + 2, i0 + 3);
  *reinterpret_cast<float4*>(coef + idx) = make_float4(c.wgt[0], c.wgt[1], c.wgt[2], c.wgt[3]);
}

// the channel's share of (d/du, d/dv): v0..v3 are the corner values, zero outside the image
__device__ __forceinline__ void slope_fma(const Corner& c, float d, float v0, float v1, float v2, float v3, float& su,
                                          float& sv) {
  const float top = (1.f - c.lx) * v0 + c.lx * v1, bot = (1.f - c.lx) * v2 + c.lx * v3;
  su = fmaf(d, (1.f - c.ly) * (v1 - v0) + c.ly * (v3 - v2), su);
  sv = fmaf(d, bot - top, sv);
}

// NHWC fp32, C % 4 == 0: one warp per pixel, lane l takes the 4-channel vectors l, l + 32, ...
__global__ void __launch_bounds__(THREADS)
sample_nhwc_kernel(const float* __restrict__ x, const float2* __restrict__ flow, const float* __restrict__ dout,
                   const float2* __restrict__ dflow_res, float2* __restrict__ dflow, uint32_t* __restrict__ keys,
                   uint32_t* __restrict__ vals, float* __restrict__ coef, int N, int H, int W, int C) {
  const int lane = threadIdx.x & 31;
  const long long M = static_cast<long long>(N) * H * W;
  const long long pix = static_cast<long long>(blockIdx.x) * WARPS + (threadIdx.x >> 5);
  if (pix >= M) return;                                      // uniform over the warp
  const int xw = static_cast<int>(pix % W);
  const int yh = static_cast<int>((pix / W) % H);
  const long long img = pix / (static_cast<long long>(W) * H) * H * W;
  const float2 f = __ldg(flow + pix);
  const Corner c = make_corners(static_cast<float>(xw) + f.x, static_cast<float>(yh) + f.y, H, W, 0);
  if (dflow) {
    const float* base = x + img * C;
    float su = 0.f, sv = 0.f;
    for (int v = lane; v < C / 4; v += 32) {
      const float4 d = __ldg(reinterpret_cast<const float4*>(dout + pix * C) + v);
      float4 val[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        val[k] = (c.in >> k & 1u) ? __ldg(reinterpret_cast<const float4*>(base + static_cast<long long>(c.off[k]) * C) + v)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
      slope_fma(c, d.x, val[0].x, val[1].x, val[2].x, val[3].x, su, sv);
      slope_fma(c, d.y, val[0].y, val[1].y, val[2].y, val[3].y, su, sv);
      slope_fma(c, d.z, val[0].z, val[1].z, val[2].z, val[3].z, su, sv);
      slope_fma(c, d.w, val[0].w, val[1].w, val[2].w, val[3].w, su, sv);
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
      su += __shfl_xor_sync(0xffffffffu, su, s);
      sv += __shfl_xor_sync(0xffffffffu, sv, s);
    }
    if (lane == 0) {
      const float2 r = dflow_res ? __ldg(dflow_res + pix) : make_float2(0.f, 0.f);
      dflow[pix] = make_float2(r.x + su, r.y + sv);
    }
  }
  if (keys && lane == 0) write_list(c, pix, img, static_cast<uint32_t>(M), keys, vals, coef);
}

// NCHW fp32 planes (the 2-channel flows), x with a batch stride: one thread per pixel, its channels in order
__global__ void __launch_bounds__(THREADS)
sample_nchw_kernel(const float* __restrict__ x, long long x_bs, const float2* __restrict__ flow,
                   const float* __restrict__ dout, const float2* __restrict__ dflow_res, float2* __restrict__ dflow,
                   uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, float* __restrict__ coef, int N, int C,
                   int H, int W) {
  const long long M = static_cast<long long>(N) * H * W;
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= M) return;
  const long long plane = static_cast<long long>(H) * W;
  const int xw = static_cast<int>(pix % W);
  const int yh = static_cast<int>((pix / W) % H);
  const long long n = pix / plane;
  const float2 f = __ldg(flow + pix);
  const Corner c = make_corners(static_cast<float>(xw) + f.x, static_cast<float>(yh) + f.y, H, W, 0);
  if (dflow) {
    const float* xb = x + n * x_bs;
    const float* db = dout + n * C * plane + (pix - n * plane);
    float su = 0.f, sv = 0.f;
    for (int ch = 0; ch < C; ++ch) {
      const float* p = xb + ch * plane;
      float v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = (c.in >> k & 1u) ? __ldg(p + c.off[k]) : 0.f;
      slope_fma(c, __ldg(db + ch * plane), v[0], v[1], v[2], v[3], su, sv);
    }
    const float2 r = dflow_res ? __ldg(dflow_res + pix) : make_float2(0.f, 0.f);
    dflow[pix] = make_float2(r.x + su, r.y + sv);
  }
  if (keys) write_list(c, pix, n * plane, static_cast<uint32_t>(M), keys, vals, coef);
}

__device__ __forceinline__ long long run_start(const uint32_t* __restrict__ keys, long long L, uint32_t d) {
  long long lo = 0, hi = L;                       // first entry with key >= d
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < d) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// dx NHWC: one thread per (destination pixel, 4 channels)
__global__ void __launch_bounds__(THREADS)
gather_nhwc_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const float* __restrict__ coef,
                   const float* __restrict__ dout, const float* __restrict__ res, float* __restrict__ dx, long long L,
                   long long M, int C) {
  const int vecs = C / 4;
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= M * vecs) return;
  const long long d = t / vecs;
  const int q = static_cast<int>(t - d * vecs);
  float4 s = res ? __ldg(reinterpret_cast<const float4*>(res + d * C) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = run_start(keys, L, static_cast<uint32_t>(d)); i < L && __ldg(keys + i) == d; ++i) {
    const uint32_t src = __ldg(vals + i);
    const float cf = __ldg(coef + src);
    const float4 a = __ldg(reinterpret_cast<const float4*>(dout + static_cast<long long>(src >> 2) * C) + q);
    s.x = fmaf(cf, a.x, s.x);
    s.y = fmaf(cf, a.y, s.y);
    s.z = fmaf(cf, a.z, s.z);
    s.w = fmaf(cf, a.w, s.w);
  }
  *reinterpret_cast<float4*>(dx + d * C + 4 * q) = s;
}

// dx NCHW (dense): one thread per destination pixel, its channels in order
__global__ void __launch_bounds__(THREADS)
gather_nchw_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const float* __restrict__ coef,
                   const float* __restrict__ dout, const float* __restrict__ res, float* __restrict__ dx, long long L,
                   long long M, int C, long long plane) {
  const long long d = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (d >= M) return;
  const long long n = d / plane, p = d - n * plane;
  const long long first = run_start(keys, L, static_cast<uint32_t>(d));
  for (int ch = 0; ch < C; ++ch) {
    const long long o = (n * C + ch) * plane + p;
    float s = res ? __ldg(res + o) : 0.f;
    for (long long i = first; i < L && __ldg(keys + i) == d; ++i) {
      const uint32_t src = __ldg(vals + i);
      const long long sp = src >> 2, sn = sp / plane;
      s = fmaf(__ldg(coef + src), __ldg(dout + (sn * C + ch) * plane + (sp - sn * plane)), s);
    }
    dx[o] = s;
  }
}

static long long list_len(long long M) { return M * 4; }

}  // namespace flow_warp_grad

long long flow_warp_backward_work_elems(int n, int h, int w) {
  return scatter::work_elems(flow_warp_grad::list_len(static_cast<long long>(n) * h * w));
}

int launch_flow_warp_backward(const float* x, long long x_bs, int nchw, const float* flow, const float* dout,
                              const float* dflow_res, float* dflow, const float* dx_res, float* dx, void* work, int n,
                              int h, int w, int c, cudaStream_t stream) {
  using namespace flow_warp_grad;
  const long long M = static_cast<long long>(n) * h * w;
  if (M == 0) return 0;
  const long long L = list_len(M);
  scatter::Work wk{};
  if (dx) wk = scatter::carve(work, L);
  const auto* fl = reinterpret_cast<const float2*>(flow);
  const auto* dr = reinterpret_cast<const float2*>(dflow_res);
  auto* df = reinterpret_cast<float2*>(dflow);
  if (nchw)
    sample_nchw_kernel<<<static_cast<unsigned>((M + THREADS - 1) / THREADS), THREADS, 0, stream>>>(
        x, x_bs, fl, dout, dr, df, wk.keys0, wk.vals0, wk.coef, n, c, h, w);
  else
    sample_nhwc_kernel<<<static_cast<unsigned>((M + WARPS - 1) / WARPS), THREADS, 0, stream>>>(
        x, fl, dout, dr, df, wk.keys0, wk.vals0, wk.coef, n, h, w, c);
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || !dx) return static_cast<int>(e);
  const uint32_t *keys = nullptr, *vals = nullptr;
  const int st = scatter::sort_pairs(wk, L, M, "flow warp backward", &keys, &vals, stream);   // keys <= M
  if (st) return st;
  if (nchw) {
    gather_nchw_kernel<<<static_cast<unsigned>((M + THREADS - 1) / THREADS), THREADS, 0, stream>>>(
        keys, vals, wk.coef, dout, dx_res, dx, L, M, c, static_cast<long long>(h) * w);
  } else {
    const long long threads = M * (c / 4);
    gather_nhwc_kernel<<<static_cast<unsigned>((threads + THREADS - 1) / THREADS), THREADS, 0, stream>>>(
        keys, vals, wk.coef, dout, dx_res, dx, L, M, c);
  }
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
