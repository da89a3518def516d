// Backward of the fused deformable alignment (dcn.cu, FUSED prologue, Cin=256, 16 deform groups, 3x3 / s1 / p1), with
// dA = dY . W16 (fp32 [M][2304], K order k = sp*16 + c, sp = g*9 + tap) computed beforehand on the linear kernel.
//
// sample_backward_kernel: one thread per (pixel, deform group), its 9 taps in order — the forward's ownership of sample
// points.  Each thread recomputes offset = max_res*fast_tanh(o) + flow.flip(1), mask = fast_sigmoid(m), the corners and
// weights under the forward's `inside` rule with the forward's instructions, and writes what is asked for:
//   * HEAD: d head (the raw conv_offset output's gradient: d offset * max_res * (1 - t^2), d mask * s * (1 - s)) and the
//     offset part of d flow_1 / d flow_2 per pixel, summed over each half's 72 sample points in a fixed order (9 taps
//     in the thread, then a shuffle tree over the half's 8 groups).  Every element has one writer: no atomics.
//   * a_hi / a_lo: the fp32 samples x mask before the forward's fp16 rounding, as the bf16 split rows of dW = dY^T A.
//   * the scatter list of dx: per (pixel, sample point, corner) a destination key ((n*16 + g)*H + y)*W + x (D = n*16*H*W
//     for corners outside the image), the source index (pixel*144 + sp)*4 + corner, and the coefficient mask * w_corner.
// The list is sorted by key with CUB's radix sort (stable, so each destination's run stays in source order), and
// gather_kernel walks every destination's run in that order: dx is the same bits on every run, no float atomics.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <climits>
#include "common.cuh"
#include "dcn_math.cuh"
#include "launch.h"
#include "scatter_sort.cuh"

namespace e2f {
namespace dcn_grad {

constexpr int CIN = 256, DG = 16, CPG = 16, TAPS = 9;
constexpr int NSP = DG * TAPS;            // 144 sample points per pixel
constexpr int KTOT = NSP * CPG;           // 2304
constexpr int HEAD_C = 3 * NSP;           // 432 raw head channels: 288 offsets ((sp, dy), (sp, dx)), 144 masks
constexpr int FLOW_C = 8;                 // d flow rows: [d flow_1 (u, v), d flow_2 (u, v), 0, 0, 0, 0]
constexpr int PIX_PER_CTA = 16;
constexpr int THREADS = PIX_PER_CTA * DG;  // 256

__device__ __forceinline__ uint32_t bf16_split_pair(float a, float b, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  lo = *reinterpret_cast<const uint32_t*>(&l);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <bool HEAD>
__global__ void __launch_bounds__(THREADS)
sample_backward_kernel(const __half* __restrict__ x, const float* __restrict__ head, const float2* __restrict__ flow1,
                       const float2* __restrict__ flow2, const float* __restrict__ da, float* __restrict__ dhead,
                       float* __restrict__ dflow, __nv_bfloat16* __restrict__ a_hi, __nv_bfloat16* __restrict__ a_lo,
                       uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, float* __restrict__ coef, int M, int H,
                       int W, float max_res) {
  const int tid = threadIdx.x, g = tid & (DG - 1);
  const long long m = static_cast<long long>(blockIdx.x) * PIX_PER_CTA + (tid >> 4);
  const bool valid = m < M;
  const long long mm = valid ? m : 0;
  const int px = static_cast<int>(mm % W);
  const int py = static_cast<int>((mm / W) % H);
  const long long n = mm / (static_cast<long long>(W) * H);
  const __half* xg = x + n * H * W * CIN + g * CPG;
  const float* hp = head + mm * HEAD_C;
  const float2 fl = __ldg((g < DG / 2 ? flow1 : flow2) + mm);
  const uint32_t sentinel = static_cast<uint32_t>(static_cast<long long>(M) * DG);     // = n*16*H*W over the batch
  const long long key_base = (n * DG + g) * H;
  float2 dfl = make_float2(0.f, 0.f);

  for (int tap = 0; tap < TAPS; ++tap) {
    const int sp = g * TAPS + tap;
    const float2 o = __ldg(reinterpret_cast<const float2*>(hp) + sp);
    const float mraw = __ldg(hp + 2 * NSP + sp);
    // the forward's prologue (dcn.cu, FUSED): offset = max_res * tanh(o) + flow.flip(1), mask = sigmoid(m)
    const float tx = dcn::fast_tanh(o.x), ty = dcn::fast_tanh(o.y);
    const float offy = fmaf(max_res, tx, fl.y);
    const float offx = fmaf(max_res, ty, fl.x);
    const float mk = dcn::fast_sigmoid(mraw);
    const int ti = tap / 3, tj = tap - ti * 3;
    const float h_im = static_cast<float>(py - 1 + ti) + offy;
    const float w_im = static_cast<float>(px - 1 + tj) + offx;
    const bool inside = valid && (h_im > -1.f) && (w_im > -1.f) && (h_im < static_cast<float>(H)) &&
                        (w_im < static_cast<float>(W));
    float acc[CPG];
#pragma unroll
    for (int c = 0; c < CPG; ++c) acc[c] = 0.f;
    float s_mask = 0.f, s_h = 0.f, s_w = 0.f;    // sum_c dA * (bilinear value, d/dh, d/dw) without the mask
    uint32_t kk[4] = {sentinel, sentinel, sentinel, sentinel};
    float cf[4] = {0.f, 0.f, 0.f, 0.f};
    if (inside) {
      const float fy = floorf(h_im), fx = floorf(w_im);
      const float ly = h_im - fy, lx = w_im - fx;
      const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
      uint4 lo[4], hi[4];
      bool in[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int dy = k >> 1, dx = k & 1;
        const int yy = y0 + dy, xx = x0 + dx;
        in[k] = (yy >= 0) && (yy < H) && (xx >= 0) && (xx < W);
        cf[k] = in[k] ? (dy ? ly : 1.f - ly) * (dx ? lx : 1.f - lx) * mk : 0.f;
        const int po = min(max(yy, 0), H - 1) * W + min(max(xx, 0), W - 1);
        const uint4* p = reinterpret_cast<const uint4*>(xg + static_cast<long long>(po) * CIN);
        lo[k] = __ldg(p);
        hi[k] = __ldg(p + 1);
        if (in[k]) kk[k] = static_cast<uint32_t>((key_base + yy) * W + xx);
      }
      float xv[4][CPG];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __half2* pl = reinterpret_cast<const __half2*>(&lo[k]);
        const __half2* ph = reinterpret_cast<const __half2*>(&hi[k]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 a = __half22float2(pl[i]);
          const float2 b = __half22float2(ph[i]);
          xv[k][2 * i] = a.x;
          xv[k][2 * i + 1] = a.y;
          xv[k][8 + 2 * i] = b.x;
          xv[k][8 + 2 * i + 1] = b.y;
        }
      }
      // the forward's sample: per channel, fmaf over the corners in order
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int c = 0; c < CPG; ++c) acc[c] = fmaf(cf[k], xv[k][c], acc[c]);
      if (HEAD) {
        float d[CPG];
        const float4* dp = reinterpret_cast<const float4*>(da + mm * KTOT + sp * CPG);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 v = __ldg(dp + i);
          d[4 * i] = v.x; d[4 * i + 1] = v.y; d[4 * i + 2] = v.z; d[4 * i + 3] = v.w;
        }
#pragma unroll
        for (int c = 0; c < CPG; ++c) {
          // corners outside the image read as zero (the floor-based bilinear form of the restatement)
          const float v0 = in[0] ? xv[0][c] : 0.f, v1 = in[1] ? xv[1][c] : 0.f;
          const float v2 = in[2] ? xv[2][c] : 0.f, v3 = in[3] ? xv[3][c] : 0.f;
          const float top = (1.f - lx) * v0 + lx * v1, bot = (1.f - lx) * v2 + lx * v3;
          s_mask = fmaf(d[c], (1.f - ly) * top + ly * bot, s_mask);
          s_h = fmaf(d[c], bot - top, s_h);
          s_w = fmaf(d[c], (1.f - ly) * (v1 - v0) + ly * (v3 - v2), s_w);
        }
      }
    }
    if (!valid) continue;
    if (a_hi) {
      uint32_t h[8], l[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) h[i] = bf16_split_pair(acc[2 * i], acc[2 * i + 1], l[i]);
      uint4* ph = reinterpret_cast<uint4*>(a_hi + mm * KTOT + sp * CPG);
      uint4* pl = reinterpret_cast<uint4*>(a_lo + mm * KTOT + sp * CPG);
      ph[0] = make_uint4(h[0], h[1], h[2], h[3]);
      ph[1] = make_uint4(h[4], h[5], h[6], h[7]);
      pl[0] = make_uint4(l[0], l[1], l[2], l[3]);
      pl[1] = make_uint4(l[4], l[5], l[6], l[7]);
    }
    if (keys) {
      const long long idx = (mm * NSP + sp) * 4;
      const uint32_t i0 = static_cast<uint32_t>(idx);
      *reinterpret_cast<uint4*>(keys + idx) = make_uint4(kk[0], kk[1], kk[2], kk[3]);
      *reinterpret_cast<uint4*>(vals + idx) = make_uint4(i0, i0 + 1, i0 + 2, i0 + 3);
      *reinterpret_cast<float4*>(coef + idx) = make_float4(cf[0], cf[1], cf[2], cf[3]);
    }
    if (HEAD) {
      const float dh = mk * s_h, dw = mk * s_w;
      *reinterpret_cast<float2*>(dhead + mm * HEAD_C + 2 * sp) =
          make_float2(dh * max_res * (1.f - tx * tx), dw * max_res * (1.f - ty * ty));
      dhead[mm * HEAD_C + 2 * NSP + sp] = s_mask * mk * (1.f - mk);
      dfl.x += dw;        // flow channel 0 (u) moves w_im
      dfl.y += dh;        // flow channel 1 (v) moves h_im
    }
  }
  if (HEAD && dflow) {
    // fixed shuffle tree over the 8 groups of each half (lanes g .. g^7 of one pixel), then half 1 to lane g = 0
#pragma unroll
    for (int s = 4; s >= 1; s >>= 1) {
      dfl.x += __shfl_xor_sync(0xffffffffu, dfl.x, s);
      dfl.y += __shfl_xor_sync(0xffffffffu, dfl.y, s);
    }
    const float ox = __shfl_down_sync(0xffffffffu, dfl.x, 8), oy = __shfl_down_sync(0xffffffffu, dfl.y, 8);
    if (valid && g == 0) {
      float4* p = reinterpret_cast<float4*>(dflow + mm * FLOW_C);
      p[0] = make_float4(dfl.x, dfl.y, ox, oy);
      p[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// dx [N][H][W][256] fp32: one thread per (destination (n, g, y, x), 4 channels); the destination's run of the sorted
// list is found by binary search and added in list (= source) order.
__global__ void __launch_bounds__(256)
gather_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const float* __restrict__ coef,
              const float* __restrict__ da, float* __restrict__ dx, long long L, long long D, int H, int W) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= D * 4) return;
  const uint32_t d = static_cast<uint32_t>(t >> 2);
  const int q = static_cast<int>(t & 3);
  long long lo = 0, hi = L;                       // first entry with key >= d
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < d) lo = mid + 1; else hi = mid;
  }
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = lo; i < L && __ldg(keys + i) == d; ++i) {
    const uint32_t src = __ldg(vals + i);
    const float c = __ldg(coef + src);
    const float4 a = __ldg(reinterpret_cast<const float4*>(da + static_cast<long long>(src >> 2) * CPG) + q);
    s.x = fmaf(c, a.x, s.x);
    s.y = fmaf(c, a.y, s.y);
    s.z = fmaf(c, a.z, s.z);
    s.w = fmaf(c, a.w, s.w);
  }
  const long long hw = static_cast<long long>(H) * W;
  const long long ng = d / hw, pix = d - ng * hw;
  const long long n = ng / DG, g = ng - n * DG;
  *reinterpret_cast<float4*>(dx + (n * hw + pix) * CIN + g * CPG + 4 * q) = s;
}

static long long list_len(long long M) { return M * NSP * 4; }

}  // namespace dcn_grad

long long dcn_backward_work_elems(int n, int h, int w) {
  using namespace dcn_grad;
  return scatter::work_elems(list_len(static_cast<long long>(n) * h * w));
}

int launch_dcn_sample_backward(const void* x, const float* head, const float* flow1, const float* flow2, const float* da,
                               float* dhead, float* dflow, void* a_hi, void* a_lo, void* work, int n, int h, int w,
                               float max_residue, cudaStream_t stream) {
  using namespace dcn_grad;
  const long long M = static_cast<long long>(n) * h * w;
  if (M == 0) return 0;
  uint32_t *keys = nullptr, *vals = nullptr;
  float* coef = nullptr;
  if (work) {
    const scatter::Work wk = scatter::carve(work, list_len(M));
    keys = wk.keys0;
    vals = wk.vals0;
    coef = wk.coef;
  }
  const unsigned blocks = static_cast<unsigned>((M + PIX_PER_CTA - 1) / PIX_PER_CTA);
  const auto* xh = static_cast<const __half*>(x);
  const auto* f1 = reinterpret_cast<const float2*>(flow1);
  const auto* f2 = reinterpret_cast<const float2*>(flow2);
  auto* ah = static_cast<__nv_bfloat16*>(a_hi);
  auto* al = static_cast<__nv_bfloat16*>(a_lo);
  const int Mi = static_cast<int>(M);
  if (dhead)
    sample_backward_kernel<true><<<blocks, THREADS, 0, stream>>>(xh, head, f1, f2, da, dhead, dflow, ah, al, keys, vals,
                                                                 coef, Mi, h, w, max_residue);
  else
    sample_backward_kernel<false><<<blocks, THREADS, 0, stream>>>(xh, head, f1, f2, nullptr, nullptr, nullptr, ah, al,
                                                                  keys, vals, coef, Mi, h, w, max_residue);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_dcn_scatter_backward(const float* da, void* work, float* dx, int n, int h, int w, cudaStream_t stream) {
  using namespace dcn_grad;
  const long long M = static_cast<long long>(n) * h * w;
  if (M == 0) return 0;
  const long long L = list_len(M), D = M * DG;
  const scatter::Work wk = scatter::carve(work, L);
  const uint32_t *keys = nullptr, *vals = nullptr;
  const int st = scatter::sort_pairs(wk, L, D, "deformable conv backward", &keys, &vals, stream);   // keys <= D
  if (st) return st;
  const long long threads = D * 4;
  gather_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(keys, vals, wk.coef,
                                                                                 da, dx, L, D, h, w);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
