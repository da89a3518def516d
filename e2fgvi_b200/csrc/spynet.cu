// SPyNet's glue (model/modules/flow_comp.py:84-169 and model/e2fgvi.py:210-234) as three small kernels, so that one
// bidirectional flow estimate is 1 + 6 x (1 + 5 convs) + 1 launches instead of ~95 (the reference issues, per level,
// an upsample, a multiply, a meshgrid + grid_sample, a cat and five convs, after 2 resizes, 2 normalisations and 10
// avg-pools):
//   spynet_pyramid      (x + 1) / 2  ->  1/4 bilinear downsample (align_corners=True, e2fgvi.py:214-218)  ->  bilinear
//                       resize to multiples of 32 (align_corners=False, flow_comp.py:152-158)  ->  (v - mean) / std  ->
//                       five 2x2 average pools (flow_comp.py:101-115), all six levels written in one pass per FRAME
//                       (the reference builds ref / supp pyramids per pair: every frame twice per direction)
//   spynet_level_input  flow_up = 2 * bilinear_x2(flow) (align_corners=True, flow_comp.py:121-126), border-mode warp of
//                       the support frame (:128-132), cat([ref, warped, flow_up]) (:127-133) written directly as the
//                       row-gapped bf16 (hi, lo) operand of the level's first 7x7 conv (window-packed K, conv.cu) plus
//                       flow_up in fp32 NHWC — the residual the level's last conv adds in its epilogue (:127)
//   spynet_final        bilinear resize back to (h, w) (align_corners=False) and the u * w / w_up, v * h / h_up rescale
//                       (flow_comp.py:160-167), written as the (b, l_t - 1, 2, h, w) flow tensors of both directions
// Index arithmetic mirrors ATen's upsample_bilinear2d / avg_pool2d so the values equal the reference's to fp32
// rounding.  Tiny, latency-bound kernels: their point is the launch count on the single-clip critical path.
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace spy {

// ATen area_pixel_compute_source_index for bilinear
__device__ __forceinline__ float src_index(float scale, int dst, bool align_corners) {
  if (align_corners) return scale * static_cast<float>(dst);
  const float s = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  return s < 0.f ? 0.f : s;
}
__host__ __device__ inline float ac_scale(int in, int out) {   // align_corners=True scale
  return out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1) : 0.f;
}

struct Lerp {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Lerp make_lerp(float src, int in) {
  Lerp t;
  t.i0 = static_cast<int>(src);
  t.i1 = t.i0 + ((t.i0 < in - 1) ? 1 : 0);
  t.l1 = src - static_cast<float>(t.i0);
  t.l0 = 1.f - t.l1;
  return t;
}

// frames: (b, t, 3, H, W) fp32 in [-1, 1] (UNIT: already in [0, 1], no (x + 1) / 2); only frames j < l_t of every clip
// are used.  One CTA = one 32 x 32 block of level 0 of one local frame; 1024 threads, thread = level-0 pixel.  pyr = the
// six levels back to back, level k holding [n][3][HU >> k][WU >> k] fp32 (n = b * l_t frames, index bi * l_t + j).
template <bool UNIT>
__global__ void __launch_bounds__(1024) spynet_pyramid_kernel(const float* __restrict__ frames, float* __restrict__ pyr,
                                                              int T, int LT, int H, int W, int h, int w, int HU, int WU,
                                                              const float* __restrict__ mean3, const float* __restrict__ std3) {
  __shared__ float lev[2][3][32][33];
  const int n = blockIdx.y;
  const int bi = n / LT, j = n - bi * LT;
  const int blocks_x = WU / 32;
  const int by = blockIdx.x / blocks_x, bx = blockIdx.x - by * blocks_x;
  const int ly = threadIdx.x >> 5, lx = threadIdx.x & 31;
  const int Y0 = by * 32 + ly, X0 = bx * 32 + lx;
  const float* fr = frames + (static_cast<long long>(bi) * T + j) * 3 * H * W;
  // level-0 pixel <- 2x2 pixels of the 1/4-size image `small` (align_corners=False) <- 2x2 full-size pixels each
  const Lerp ry = make_lerp(src_index(static_cast<float>(h) / static_cast<float>(HU), Y0, false), h);
  const Lerp rx = make_lerp(src_index(static_cast<float>(w) / static_cast<float>(WU), X0, false), w);
  const float sc_y = ac_scale(H, h), sc_x = ac_scale(W, w);
  const int sy[2] = {ry.i0, ry.i1}, sx[2] = {rx.i0, rx.i1};
  Lerp dy[2], dx[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    dy[a] = make_lerp(src_index(sc_y, sy[a], true), H);
    dx[a] = make_lerp(src_index(sc_x, sx[a], true), W);
  }
  const float mean[3] = {__ldg(mean3), __ldg(mean3 + 1), __ldg(mean3 + 2)};
  const float stdv[3] = {__ldg(std3), __ldg(std3 + 1), __ldg(std3 + 2)};
  const long long plane = static_cast<long long>(H) * W;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* p = fr + c * plane;
    float sm[2][2];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
      for (int b2 = 0; b2 < 2; ++b2) {
        // (x + 1) / 2 of e2fgvi.py:247 (UNIT: the [0, 1] value as given), then the align_corners=True bilinear sample
        float v00 = __ldg(p + static_cast<long long>(dy[a].i0) * W + dx[b2].i0);
        float v01 = __ldg(p + static_cast<long long>(dy[a].i0) * W + dx[b2].i1);
        float v10 = __ldg(p + static_cast<long long>(dy[a].i1) * W + dx[b2].i0);
        float v11 = __ldg(p + static_cast<long long>(dy[a].i1) * W + dx[b2].i1);
        if constexpr (!UNIT) {
          v00 = (v00 + 1.f) / 2.f;
          v01 = (v01 + 1.f) / 2.f;
          v10 = (v10 + 1.f) / 2.f;
          v11 = (v11 + 1.f) / 2.f;
        }
        sm[a][b2] = dy[a].l0 * (dx[b2].l0 * v00 + dx[b2].l1 * v01) + dy[a].l1 * (dx[b2].l0 * v10 + dx[b2].l1 * v11);
      }
    }
    const float v = ry.l0 * (rx.l0 * sm[0][0] + rx.l1 * sm[0][1]) + ry.l1 * (rx.l0 * sm[1][0] + rx.l1 * sm[1][1]);
    const float nv = (v - mean[c]) / stdv[c];
    lev[0][c][ly][lx] = nv;
    pyr[(static_cast<long long>(n) * 3 + c) * HU * WU + static_cast<long long>(Y0) * WU + X0] = nv;
  }
  long long off = static_cast<long long>(gridDim.y) * 3 * HU * WU;     // start of level 1
  int cur = 0;
#pragma unroll 1
  for (int k = 1; k <= 5; ++k) {
    __syncthreads();
    const int side = 32 >> k, hk = HU >> k, wk = WU >> k;
    if (ly < side && lx < side) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // ATen avg_pool2d: running sum in (kh, kw) order, then / 4
        const float s = ((lev[cur][c][2 * ly][2 * lx] + lev[cur][c][2 * ly][2 * lx + 1]) + lev[cur][c][2 * ly + 1][2 * lx]) +
                        lev[cur][c][2 * ly + 1][2 * lx + 1];
        const float v = s / 4.f;
        lev[cur ^ 1][c][ly][lx] = v;
        pyr[off + (static_cast<long long>(n) * 3 + c) * hk * wk + static_cast<long long>(by * side + ly) * wk + bx * side + lx] = v;
      }
    }
    off += static_cast<long long>(gridDim.y) * 3 * hk * wk;
    cur ^= 1;
  }
}

// One thread per pixel SLOT of the row-gapped operand (lead zero pixels in front of every row + tail), like
// pack_rows_kernel (conv.cu).  img: level image [n][3][hk][wk]; prev: flow of the coarser level [P][hk/2][wk/2][2] fp32
// or null (level 0: zero flow).  P = 2 * b * (LT - 1) pairs: direction-major, then clip, then j; forward pairs use
// (ref, supp) = frames (j, j + 1), backward pairs (j + 1, j)  (e2fgvi.py:221-229).
__global__ void __launch_bounds__(256) spynet_level_input_kernel(const float* __restrict__ img, const float* __restrict__ prev,
                                                                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                                                 float* __restrict__ flow_up, int P, int B, int LT, int hk,
                                                                 int wk, int lead, int pitch, int tail) {
  const long long total = static_cast<long long>(P) * hk * pitch + tail;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long row = i / pitch;
  const int x = static_cast<int>(i - row * pitch) - lead;
  float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (row < static_cast<long long>(P) * hk && x >= 0 && x < wk) {
    const int p = static_cast<int>(row / hk), y = static_cast<int>(row - static_cast<long long>(p) * hk);
    const int per_dir = B * (LT - 1);
    const int dir = p / per_dir, q = p - dir * per_dir;
    const int bi = q / (LT - 1), j = q - bi * (LT - 1);
    const int ref_n = bi * LT + (dir ? j + 1 : j), sup_n = bi * LT + (dir ? j : j + 1);
    float fu = 0.f, fv = 0.f;
    if (prev) {
      // F.interpolate(flow, scale_factor=2, bilinear, align_corners=True) * 2.0
      const int hp = hk >> 1, wp = wk >> 1;
      const Lerp ty = make_lerp(src_index(ac_scale(hp, hk), y, true), hp);
      const Lerp tx = make_lerp(src_index(ac_scale(wp, wk), x, true), wp);
      const float2* pf = reinterpret_cast<const float2*>(prev) + static_cast<long long>(p) * hp * wp;
      const float2 a = __ldg(pf + ty.i0 * wp + tx.i0), b2 = __ldg(pf + ty.i0 * wp + tx.i1);
      const float2 c = __ldg(pf + ty.i1 * wp + tx.i0), d = __ldg(pf + ty.i1 * wp + tx.i1);
      fu = (ty.l0 * (tx.l0 * a.x + tx.l1 * b2.x) + ty.l1 * (tx.l0 * c.x + tx.l1 * d.x)) * 2.0f;
      fv = (ty.l0 * (tx.l0 * a.y + tx.l1 * b2.y) + ty.l1 * (tx.l0 * c.y + tx.l1 * d.y)) * 2.0f;
    }
    // border-mode warp of the support image (flow_warp(..., padding_mode='border'), flow_comp.py:128-132)
    float px = fminf(fmaxf(static_cast<float>(x) + fu, 0.f), static_cast<float>(wk - 1));
    float py = fminf(fmaxf(static_cast<float>(y) + fv, 0.f), static_cast<float>(hk - 1));
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float lx = px - fx0, ly = py - fy0;
    const int x0 = static_cast<int>(fx0), y0 = static_cast<int>(fy0);
    const int x1 = min(x0 + 1, wk - 1), y1 = min(y0 + 1, hk - 1);
    // a corner beyond the last row / column only ever carries weight 0 after the clamp (lx == 0 or ly == 0 there)
    const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
    const long long plane = static_cast<long long>(hk) * wk;
    const float* rp = img + static_cast<long long>(ref_n) * 3 * plane + static_cast<long long>(y) * wk + x;
    const float* sp = img + static_cast<long long>(sup_n) * 3 * plane;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      f[c] = __ldg(rp + c * plane);
      const float* s = sp + c * plane;
      float acc = 0.f;
      acc = fmaf(w00, __ldg(s + y0 * wk + x0), acc);
      acc = fmaf(w01, __ldg(s + y0 * wk + x1), acc);
      acc = fmaf(w10, __ldg(s + y1 * wk + x0), acc);
      acc = fmaf(w11, __ldg(s + y1 * wk + x1), acc);
      f[3 + c] = acc;
    }
    f[6] = fu;
    f[7] = fv;
    reinterpret_cast<float2*>(flow_up)[(static_cast<long long>(p) * hk + y) * wk + x] = make_float2(fu, fv);
  }
  uint32_t hp[4], lp[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const __nv_bfloat162 hb = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
    const float2 hf = __bfloat1622float2(hb);
    const __nv_bfloat162 lb = __floats2bfloat162_rn(f[2 * k] - hf.x, f[2 * k + 1] - hf.y);
    hp[k] = *reinterpret_cast<const uint32_t*>(&hb);
    lp[k] = *reinterpret_cast<const uint32_t*>(&lb);
  }
  *reinterpret_cast<uint4*>(hi + i * 8) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
  *reinterpret_cast<uint4*>(lo + i * 8) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
}

// flow: [P][HU][WU][2] fp32 (level 5).  out_fwd / out_bwd: (b, LT - 1, 2, h, w) fp32.
__global__ void __launch_bounds__(256) spynet_final_kernel(const float* __restrict__ flow, float* __restrict__ out_fwd,
                                                           float* __restrict__ out_bwd, int P, int h, int w, int HU, int WU) {
  const long long total = static_cast<long long>(P) * h * w;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = static_cast<int>(i % w), y = static_cast<int>((i / w) % h);
  const int p = static_cast<int>(i / (static_cast<long long>(w) * h));
  const Lerp ty = make_lerp(src_index(static_cast<float>(HU) / static_cast<float>(h), y, false), HU);
  const Lerp tx = make_lerp(src_index(static_cast<float>(WU) / static_cast<float>(w), x, false), WU);
  const float2* pf = reinterpret_cast<const float2*>(flow) + static_cast<long long>(p) * HU * WU;
  const float2 a = __ldg(pf + ty.i0 * WU + tx.i0), b = __ldg(pf + ty.i0 * WU + tx.i1);
  const float2 c = __ldg(pf + ty.i1 * WU + tx.i0), d = __ldg(pf + ty.i1 * WU + tx.i1);
  const float u = ty.l0 * (tx.l0 * a.x + tx.l1 * b.x) + ty.l1 * (tx.l0 * c.x + tx.l1 * d.x);
  const float v = ty.l0 * (tx.l0 * a.y + tx.l1 * b.y) + ty.l1 * (tx.l0 * c.y + tx.l1 * d.y);
  const int half = P / 2;
  float* o = (p < half ? out_fwd + static_cast<long long>(p) * 2 * h * w : out_bwd + static_cast<long long>(p - half) * 2 * h * w);
  o[static_cast<long long>(y) * w + x] = u * (static_cast<float>(w) / static_cast<float>(WU));
  o[static_cast<long long>(h) * w + static_cast<long long>(y) * w + x] = v * (static_cast<float>(h) / static_cast<float>(HU));
}

// ----------------------------------------------------------------------------------------------------------- backward
// Pair p's (ref, supp) frame indices (see spynet_level_input_kernel).
__device__ __forceinline__ int support_frame(int p, int B, int LT) {
  const int per_dir = B * (LT - 1);
  const int dir = p / per_dir, q = p - dir * per_dir;
  const int bi = q / (LT - 1), j = q - bi * (LT - 1);
  return bi * LT + (dir ? j : j + 1);
}

// Gradient reaching flow_up at fine pixel (p, y, x): the residual's dflow, the flow_up channels 6..7 of the conv input's
// gradient d_in, and the border-mode warp's coordinate gradient from channels 3..5, with torch's grid_sampler_2d backward
// conventions (a coordinate at or beyond the border gets zero gradient in that axis; out-of-range corners read 0).
__device__ __forceinline__ float2 flow_up_grad(const float* __restrict__ d_in, const float* __restrict__ dflow,
                                              const float* __restrict__ sp, const float* __restrict__ flow_up, long long pix,
                                              int y, int x, int hk, int wk) {
  const float2 fl = __ldg(reinterpret_cast<const float2*>(flow_up) + pix);
  const float2 df = __ldg(reinterpret_cast<const float2*>(dflow) + pix);
  const float* d = d_in + pix * 8;
  float gu = df.x + __ldg(d + 6), gv = df.y + __ldg(d + 7);
  const float ix = static_cast<float>(x) + fl.x, iy = static_cast<float>(y) + fl.y;
  const bool in_x = ix > 0.f && ix < static_cast<float>(wk - 1), in_y = iy > 0.f && iy < static_cast<float>(hk - 1);
  if (in_x || in_y) {
    const float px = fminf(fmaxf(ix, 0.f), static_cast<float>(wk - 1)), py = fminf(fmaxf(iy, 0.f), static_cast<float>(hk - 1));
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float lx = px - fx0, ly = py - fy0;
    const int x0 = static_cast<int>(fx0), y0 = static_cast<int>(fy0);
    const bool x1_ok = x0 + 1 < wk, y1_ok = y0 + 1 < hk;
    const long long plane = static_cast<long long>(hk) * wk;
    float gix = 0.f, giy = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* s = sp + c * plane;
      const float g = __ldg(d + 3 + c);
      const float v00 = __ldg(s + y0 * wk + x0);
      const float v01 = x1_ok ? __ldg(s + y0 * wk + x0 + 1) : 0.f;
      const float v10 = y1_ok ? __ldg(s + (y0 + 1) * wk + x0) : 0.f;
      const float v11 = (x1_ok && y1_ok) ? __ldg(s + (y0 + 1) * wk + x0 + 1) : 0.f;
      gix = fmaf(g, (1.f - ly) * (v01 - v00) + ly * (v11 - v10), gix);
      giy = fmaf(g, (1.f - lx) * (v10 - v00) + lx * (v11 - v01), giy);
    }
    if (in_x) gu += gix;
    if (in_y) gv += giy;
  }
  return make_float2(gu, gv);
}

// Adjoint of spynet_level_input_kernel with respect to prev (the coarser level's flow), as a gather: thread = coarse
// pixel (p, py, px); it visits the fine pixels whose x2 upsample (align_corners=True) reads it, in a fixed order, and adds
// 2 * weight * flow_up_grad.  No atomics: deterministic.
__global__ void __launch_bounds__(256) spynet_level_input_backward_kernel(const float* __restrict__ d_in,
                                                                          const float* __restrict__ dflow,
                                                                          const float* __restrict__ img,
                                                                          const float* __restrict__ flow_up,
                                                                          float* __restrict__ dprev, int P, int B, int LT,
                                                                          int hk, int wk) {
  const int hp = hk >> 1, wp = wk >> 1;
  const long long total = static_cast<long long>(P) * hp * wp;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int px = static_cast<int>(i % wp), py = static_cast<int>((i / wp) % hp);
  const int p = static_cast<int>(i / (static_cast<long long>(wp) * hp));
  const float* sp = img + static_cast<long long>(support_frame(p, B, LT)) * 3 * hk * wk;
  const float sy = ac_scale(hp, hk), sx = ac_scale(wp, wk);
  // fine rows / columns whose lerp taps can include py / px: src = y (hp - 1) / (hk - 1) < y / 2
  const int y_lo = max(0, 2 * py - 3), y_hi = min(hk - 1, 2 * py + 4);
  const int x_lo = max(0, 2 * px - 3), x_hi = min(wk - 1, 2 * px + 4);
  float au = 0.f, av = 0.f;
  for (int y = y_lo; y <= y_hi; ++y) {
    const Lerp ty = make_lerp(src_index(sy, y, true), hp);
    const float wy = (ty.i0 == py ? ty.l0 : 0.f) + (ty.i1 == py ? ty.l1 : 0.f);
    if (wy == 0.f) continue;
    for (int x = x_lo; x <= x_hi; ++x) {
      const Lerp tx = make_lerp(src_index(sx, x, true), wp);
      const float wx = (tx.i0 == px ? tx.l0 : 0.f) + (tx.i1 == px ? tx.l1 : 0.f);
      if (wx == 0.f) continue;
      const float2 g = flow_up_grad(d_in, dflow, sp, flow_up, (static_cast<long long>(p) * hk + y) * wk + x, y, x, hk, wk);
      const float w2 = 2.0f * wy * wx;
      au = fmaf(w2, g.x, au);
      av = fmaf(w2, g.y, av);
    }
  }
  reinterpret_cast<float2*>(dprev)[i] = make_float2(au, av);
}

// Adjoint of spynet_final_kernel: thread = level-5 flow pixel (p, Y, X); gathers, in a fixed order, the output pixels
// whose align_corners=False resize reads it, times the u / v rescale.
__global__ void __launch_bounds__(256) spynet_final_backward_kernel(const float* __restrict__ d_fwd, const float* __restrict__ d_bwd,
                                                                    float* __restrict__ dflow, int P, int h, int w, int HU, int WU) {
  const long long total = static_cast<long long>(P) * HU * WU;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = static_cast<int>(i % WU), Y = static_cast<int>((i / WU) % HU);
  const int p = static_cast<int>(i / (static_cast<long long>(WU) * HU));
  const int half = P / 2;
  const float* g = p < half ? d_fwd + static_cast<long long>(p) * 2 * h * w : d_bwd + static_cast<long long>(p - half) * 2 * h * w;
  const float scy = static_cast<float>(HU) / static_cast<float>(h), scx = static_cast<float>(WU) / static_cast<float>(w);
  // output rows whose source index lies in [Y - 1, Y + 1): the scale HU / h is >= 1
  const int y_lo = max(0, (Y - 1) * h / HU - 1), y_hi = min(h - 1, ((Y + 1) * h + HU - 1) / HU + 1);
  const int x_lo = max(0, (X - 1) * w / WU - 1), x_hi = min(w - 1, ((X + 1) * w + WU - 1) / WU + 1);
  float au = 0.f, av = 0.f;
  for (int y = y_lo; y <= y_hi; ++y) {
    const Lerp ty = make_lerp(src_index(scy, y, false), HU);
    const float wy = (ty.i0 == Y ? ty.l0 : 0.f) + (ty.i1 == Y ? ty.l1 : 0.f);
    if (wy == 0.f) continue;
    for (int x = x_lo; x <= x_hi; ++x) {
      const Lerp tx = make_lerp(src_index(scx, x, false), WU);
      const float wx = (tx.i0 == X ? tx.l0 : 0.f) + (tx.i1 == X ? tx.l1 : 0.f);
      if (wx == 0.f) continue;
      const float wt = wy * wx;
      au = fmaf(wt, __ldg(g + static_cast<long long>(y) * w + x), au);
      av = fmaf(wt, __ldg(g + static_cast<long long>(h) * w + static_cast<long long>(y) * w + x), av);
    }
  }
  reinterpret_cast<float2*>(dflow)[i] =
      make_float2(au * (static_cast<float>(w) / static_cast<float>(WU)), av * (static_cast<float>(h) / static_cast<float>(HU)));
}

}  // namespace spy

int launch_spynet_pyramid(const float* frames, float* pyr, int b, int t, int lt, int H, int W, int h, int w, int hu, int wu,
                          const float* mean3, const float* std3, cudaStream_t stream) {
  if (b == 0) return 0;
  const dim3 grid((hu / 32) * (wu / 32), b * lt);
  spy::spynet_pyramid_kernel<false><<<grid, 1024, 0, stream>>>(frames, pyr, t, lt, H, W, h, w, hu, wu, mean3, std3);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_spynet_pyramid_unit(const float* frames, float* pyr, int b, int t, int lt, int H, int W, int h, int w, int hu,
                               int wu, const float* mean3, const float* std3, cudaStream_t stream) {
  if (b == 0) return 0;
  const dim3 grid((hu / 32) * (wu / 32), b * lt);
  spy::spynet_pyramid_kernel<true><<<grid, 1024, 0, stream>>>(frames, pyr, t, lt, H, W, h, w, hu, wu, mean3, std3);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_spynet_level_input(const float* img, const float* prev, void* hi, void* lo, float* flow_up, int b, int lt, int hk,
                              int wk, int lead, cudaStream_t stream) {
  const int P = 2 * b * (lt - 1);
  if (P == 0) return 0;
  const int pitch = conv_rows_pitch(wk, lead, 8), tail = conv_rows_tail(lead, 8);
  const long long total = static_cast<long long>(P) * hk * pitch + tail;
  spy::spynet_level_input_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      img, prev, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), flow_up, P, b, lt, hk, wk, lead, pitch, tail);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_spynet_final(const float* flow, float* out_fwd, float* out_bwd, int b, int lt, int h, int w, int hu, int wu,
                        cudaStream_t stream) {
  const int P = 2 * b * (lt - 1);
  if (P == 0) return 0;
  const long long total = static_cast<long long>(P) * h * w;
  spy::spynet_final_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(flow, out_fwd, out_bwd, P, h, w, hu, wu);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_spynet_level_input_backward(const float* d_in, const float* dflow, const float* img, const float* flow_up,
                                       float* dprev, int b, int lt, int hk, int wk, cudaStream_t stream) {
  const int P = 2 * b * (lt - 1);
  if (P == 0) return 0;
  const long long total = static_cast<long long>(P) * (hk / 2) * (wk / 2);
  spy::spynet_level_input_backward_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      d_in, dflow, img, flow_up, dprev, P, b, lt, hk, wk);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_spynet_final_backward(const float* d_fwd, const float* d_bwd, float* dflow, int b, int lt, int h, int w, int hu,
                                 int wu, cudaStream_t stream) {
  const int P = 2 * b * (lt - 1);
  if (P == 0) return 0;
  const long long total = static_cast<long long>(P) * hu * wu;
  spy::spynet_final_backward_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(d_fwd, d_bwd, dflow, P, h,
                                                                                                     w, hu, wu);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
