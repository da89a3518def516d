// Producer-side fusions that emit the bf16 (hi, lo) operand pairs of the bf16x3 GEMM / conv kernels directly:
//   upsample2x_split : F.interpolate(scale_factor=2, bilinear, align_corners=True) of e2fgvi.py:125-129 on NHWC fp32,
//                      written as the split operand of the following conv (the 4x larger fp32 tensor never exists)
//   layernorm_split  : nn.LayerNorm over the last dim (tfocal_transformer.py:470,533) -> fp32 and/or split output
// HBM-bound elementwise kernels; algorithmic bytes = input read + outputs written.
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {

__device__ __forceinline__ void split_store8(const float (&f)[8], __nv_bfloat16* hi, __nv_bfloat16* lo) {
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

// read-only load of 8 consecutive, 32-byte aligned floats (two 128-bit loads)
__device__ __forceinline__ void ldg256_f32(const float4* p, float (&v)[8]) {
  const float4 a = __ldg(p), b = __ldg(p + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// one thread per (output pixel, 8 channels); source index arithmetic mirrors ATen's upsample_bilinear2d.
// grid = (x blocks, output row, image): no 64-bit div / mod chain per thread (the first version decoded a flat 64-bit
// index: ~45 % of its instructions, 3.1 TB/s)
__global__ void __launch_bounds__(256) upsample2x_split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                                                               __nv_bfloat16* __restrict__ lo, int N, int H, int W, int C,
                                                               float rh, float rw) {
  const int OH = 2 * H, OW = 2 * W, V = C / 8;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= OW * V) return;
  const int ox = t / V, v = t - ox * V;
  const int oy = blockIdx.y;
  const long long n = blockIdx.z;
  const long long pix = (n * OH + oy) * OW + ox;
  const float sy = rh * oy, sx = rw * ox;                     // rh, rw: (in - 1) / (out - 1) in fp32, as ATen computes them
  const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
  const int y1 = y0 + ((y0 < H - 1) ? 1 : 0), x1 = x0 + ((x0 < W - 1) ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const float* base = x + n * H * W * C + v * 8;
  const float4* p00 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y0) * W + x0) * C);
  const float4* p01 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y0) * W + x1) * C);
  const float4* p10 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y1) * W + x0) * C);
  const float4* p11 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y1) * W + x1) * C);
  // one 256-bit request per corner (8 fp32 channels = 32 aligned bytes): ncu showed the kernel L1-bound (l1tex 94-96 %)
  // with two LDG.128 per corner
  float a[8], b[8], c[8], d[8];
  ldg256_f32(p00, a);
  ldg256_f32(p01, b);
  ldg256_f32(p10, c);
  ldg256_f32(p11, d);
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = hy * (hx * a[i] + lx * b[i]) + ly * (hx * c[i] + lx * d[i]);
  const long long o = pix * C + v * 8;
  split_store8(f, hi + o, lo + o);
}

// one warp per PAIR of rows of C = 32 * PER_LANE floats (C = 512 -> 16 per lane and row): the loads of both rows are
// issued before the first reduction (twice the bytes in flight per warp); two-pass mean / variance in registers
template <int PER_LANE>
__global__ void __launch_bounds__(256) layernorm_split_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, float* __restrict__ out,
                                                              __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                                              long long rows, float eps) {
  constexpr int C = 32 * PER_LANE, R = 2;
  const long long row0 = (static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R;
  if (row0 >= rows) return;
  const int lane = threadIdx.x & 31;
  float v[R][PER_LANE];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const bool ok = row0 + r < rows;
    const float* xr = x + (row0 + (ok ? r : 0)) * C;
#pragma unroll
    for (int j = 0; j < PER_LANE / 8; ++j) {        // lane owns 8 consecutive floats per 256-float segment
      const float4 a = __ldg(reinterpret_cast<const float4*>(xr + j * 256 + lane * 8));
      const float4 b = __ldg(reinterpret_cast<const float4*>(xr + j * 256 + lane * 8) + 1);
      v[r][8 * j + 0] = a.x; v[r][8 * j + 1] = a.y; v[r][8 * j + 2] = a.z; v[r][8 * j + 3] = a.w;
      v[r][8 * j + 4] = b.x; v[r][8 * j + 5] = b.y; v[r][8 * j + 6] = b.z; v[r][8 * j + 7] = b.w;
    }
  }
  float g[PER_LANE], bt[PER_LANE];
#pragma unroll
  for (int j = 0; j < PER_LANE / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      g[8 * j + e] = __ldg(gamma + j * 256 + lane * 8 + e);
      bt[8 * j + e] = __ldg(beta + j * 256 + lane * 8 + e);
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (row0 + r >= rows) break;
    const long long row = row0 + r;
    float sum = 0.f;
#pragma unroll
    for (int e = 0; e < PER_LANE; ++e) sum += v[r][e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * (1.0f / C);
    float sq = 0.f;
#pragma unroll
    for (int e = 0; e < PER_LANE; ++e) {
      const float d = v[r][e] - mean;
      sq = fmaf(d, d, sq);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq * (1.0f / C) + eps);
#pragma unroll
    for (int j = 0; j < PER_LANE / 8; ++j) {
      const int c0 = j * 256 + lane * 8;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = (v[r][8 * j + e] - mean) * rstd * g[8 * j + e] + bt[8 * j + e];
      if (out) {
        float4* d4 = reinterpret_cast<float4*>(out + row * C + c0);
        d4[0] = make_float4(f[0], f[1], f[2], f[3]);
        d4[1] = make_float4(f[4], f[5], f[6], f[7]);
      }
      if (hi) split_store8(f, hi + row * C + c0, lo + row * C + c0);
    }
  }
}

// LayerNorm + FOCAL WINDOW POOLING in one pass (tfocal_transformer.py:470 norm1 + :508-516 pool_layers[0]): one CTA per
// (frame, window); each warp normalises whole token rows (512 channels, 16 per lane) and, with the normalised fp32
// values still IN REGISTERS, accumulates its share of the window's pooled token  sum_tok w[tok] * LN(x[tok])  per channel;
// the 8 per-warp partial rows are reduced through 16 KB of shared memory.  Outputs: the bf16 (hi, lo) split of the
// normalised tokens, rows [0, BT*H*W), and of the pooled tokens, rows [BT*H*W, +BT*nW) of the SAME buffers, ordered
// (bt, wi, wj) — so ONE qkv GEMM serves tokens and pooled tokens and the standalone pool / pooled-qkv launches are gone.
template <int PER_LANE>
__global__ void __launch_bounds__(256) layernorm_pool_split_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                                   const float* __restrict__ beta,
                                                                   const float* __restrict__ pool_w,
                                                                   const float* __restrict__ pool_b,
                                                                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                                                   int H, int W, int wh, int ww, long long rows, float eps) {
  constexpr int C = 32 * PER_LANE;
  __shared__ float red[8][C];
  const int nww = W / ww, nwh = H / wh;
  const int win = blockIdx.x, bt = blockIdx.y;
  const int wi = win / nww, wj = win - wi * nww;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g[PER_LANE], bt_[PER_LANE], acc[PER_LANE];
#pragma unroll
  for (int j = 0; j < PER_LANE / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      g[8 * j + e] = __ldg(gamma + j * 256 + lane * 8 + e);
      bt_[8 * j + e] = __ldg(beta + j * 256 + lane * 8 + e);
      acc[8 * j + e] = 0.f;
    }
  }
  const int ntok = wh * ww;
  for (int tok = warp; tok < ntok; tok += 8) {
    const int r = tok / ww, q = tok - r * ww;
    const long long row = (static_cast<long long>(bt) * H + wi * wh + r) * W + wj * ww + q;
    const float* xr = x + row * C;
    float v[PER_LANE];
#pragma unroll
    for (int j = 0; j < PER_LANE / 8; ++j) {        // lane owns 8 consecutive floats per 256-float segment
      const float4 a = __ldg(reinterpret_cast<const float4*>(xr + j * 256 + lane * 8));
      const float4 b = __ldg(reinterpret_cast<const float4*>(xr + j * 256 + lane * 8) + 1);
      v[8 * j + 0] = a.x; v[8 * j + 1] = a.y; v[8 * j + 2] = a.z; v[8 * j + 3] = a.w;
      v[8 * j + 4] = b.x; v[8 * j + 5] = b.y; v[8 * j + 6] = b.z; v[8 * j + 7] = b.w;
    }
    float sum = 0.f;
#pragma unroll
    for (int e = 0; e < PER_LANE; ++e) sum += v[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * (1.0f / C);
    float sq = 0.f;
#pragma unroll
    for (int e = 0; e < PER_LANE; ++e) {
      const float d = v[e] - mean;
      sq = fmaf(d, d, sq);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq * (1.0f / C) + eps);
    const float wt = __ldg(pool_w + tok);
#pragma unroll
    for (int j = 0; j < PER_LANE / 8; ++j) {
      const int c0 = j * 256 + lane * 8;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        f[e] = (v[8 * j + e] - mean) * rstd * g[8 * j + e] + bt_[8 * j + e];
        acc[8 * j + e] = fmaf(wt, f[e], acc[8 * j + e]);
      }
      split_store8(f, hi + row * C + c0, lo + row * C + c0);
    }
  }
#pragma unroll
  for (int j = 0; j < PER_LANE / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 8; ++e) red[warp][j * 256 + lane * 8 + e] = acc[8 * j + e];
  }
  __syncthreads();
  // pooled token: fixed summation order over the 8 warps (deterministic); 64 threads x 8 channels
  if (threadIdx.x < C / 8) {
    const int c0 = threadIdx.x * 8;
    const float b0 = pool_b ? __ldg(pool_b) : 0.f;
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float t = b0;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += red[k][c0 + e];
      f[e] = t;
    }
    const long long prow = rows + (static_cast<long long>(bt) * nwh + wi) * nww + wj;
    split_store8(f, hi + prow * C + c0, lo + prow * C + c0);
  }
}

// Window pooling of the focal attention's coarse level (pool_layers[0] = nn.Linear(wh*ww, 1) applied across the tokens
// of each window, per channel; tfocal_transformer.py:508-516):
//   out[bt][wi][wj][c] = bias + sum_{r,q} x[bt][wi*wh + r][wj*ww + q][c] * weight[r*ww + q]
// x comes as the bf16 (hi, lo) pair LayerNorm already wrote for the qkv Linear, so the fp32 copy of the normed tokens
// is never materialised; the result goes out as the (hi, lo) operand pair of the pooled qkv Linear (and/or fp32).
// Block = one window x 64 channel-octets x wh window rows (threadIdx.y); rows reduced through shared memory.
__global__ void __launch_bounds__(512) window_pool_kernel(const __nv_bfloat16* __restrict__ xh,
                                                          const __nv_bfloat16* __restrict__ xl,
                                                          const float* __restrict__ weight, const float* __restrict__ bias,
                                                          float* __restrict__ out, __nv_bfloat16* __restrict__ out_hi,
                                                          __nv_bfloat16* __restrict__ out_lo, int H, int W, int C, int wh,
                                                          int ww) {
  extern __shared__ float red[];                   // [wh][C]
  const int nww = W / ww, nwh = H / wh;
  const int win = blockIdx.x, bt = blockIdx.y;
  const int wi = win / nww, wj = win - wi * nww;
  const int r = threadIdx.y;
  for (int c0 = threadIdx.x * 8; c0 < C; c0 += blockDim.x * 8) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const size_t row0 = ((static_cast<size_t>(bt) * H + wi * wh + r) * W + wj * ww) * C + c0;
    for (int q = 0; q < ww; ++q) {
      const float wt = __ldg(weight + r * ww + q);
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(xh + row0 + static_cast<size_t>(q) * C));
      const uint4 b = __ldg(reinterpret_cast<const uint4*>(xl + row0 + static_cast<size_t>(q) * C));
      const uint32_t ah[4] = {a.x, a.y, a.z, a.w}, bl[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 fh = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ah[e]));
        const float2 fl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&bl[e]));
        acc[2 * e] = fmaf(fh.x + fl.x, wt, acc[2 * e]);
        acc[2 * e + 1] = fmaf(fh.y + fl.y, wt, acc[2 * e + 1]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[r * C + c0 + e] = acc[e];
  }
  __syncthreads();
  if (r == 0) {
    const float b0 = bias ? __ldg(bias) : 0.f;
    for (int c0 = threadIdx.x * 8; c0 < C; c0 += blockDim.x * 8) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float t = b0;
        for (int k = 0; k < wh; ++k) t += red[k * C + c0 + e];
        f[e] = t;
      }
      const size_t o = ((static_cast<size_t>(bt) * nwh + wi) * nww + wj) * C + c0;
      if (out) {
        float4* d4 = reinterpret_cast<float4*>(out + o);
        d4[0] = make_float4(f[0], f[1], f[2], f[3]);
        d4[1] = make_float4(f[4], f[5], f[6], f[7]);
      }
      if (out_hi) split_store8(f, out_hi + o, out_lo + o);
    }
  }
}

int launch_window_pool(const void* xh, const void* xl, const float* weight, const float* bias, float* out, void* out_hi,
                       void* out_lo, int bt, int h, int w, int c, int wh, int ww, cudaStream_t stream) {
  if (bt == 0) return 0;
  const dim3 grid((h / wh) * (w / ww), bt), block(c / 8 < 64 ? c / 8 : 64, wh);
  window_pool_kernel<<<grid, block, static_cast<size_t>(wh) * c * sizeof(float), stream>>>(
      static_cast<const __nv_bfloat16*>(xh), static_cast<const __nv_bfloat16*>(xl), weight, bias, out,
      static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), h, w, c, wh, ww);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_layernorm_pool_split(const float* x, const float* gamma, const float* beta, const float* pool_w,
                                const float* pool_b, void* hi, void* lo, int bt, int h, int w, int c, int wh, int ww,
                                float eps, cudaStream_t stream) {
  if (bt == 0) return 0;
  if (c != 512) {
    set_error("layernorm_pool_split is specialised for 512 channels (got %d)", c);
    return -2;
  }
  const dim3 grid((h / wh) * (w / ww), bt);
  layernorm_pool_split_kernel<16><<<grid, 256, 0, stream>>>(x, gamma, beta, pool_w, pool_b, static_cast<__nv_bfloat16*>(hi),
                                                            static_cast<__nv_bfloat16*>(lo), h, w, wh, ww,
                                                            static_cast<long long>(bt) * h * w, eps);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_upsample2x_split(const float* x, void* hi, void* lo, int n, int h, int w, int c, cudaStream_t stream) {
  const long long total = static_cast<long long>(n) * 4 * h * w * (c / 8);
  if (total == 0) return 0;
  if (n > 65535 || 2 * h > 65535) {
    set_error("upsample2x_split: at most 65535 images / output rows per launch (got %d, %d)", n, 2 * h);
    return -2;
  }
  const int threads = 256, row_threads = 2 * w * (c / 8);
  const dim3 grid((row_threads + threads - 1) / threads, 2 * h, n);
  const float rh = (2 * h > 1) ? static_cast<float>(h - 1) / static_cast<float>(2 * h - 1) : 0.f;
  const float rw = (2 * w > 1) ? static_cast<float>(w - 1) / static_cast<float>(2 * w - 1) : 0.f;
  upsample2x_split_kernel<<<grid, threads, 0, stream>>>(x, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), n, h,
                                                       w, c, rh, rw);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_layernorm_split(const float* x, const float* gamma, const float* beta, float* out, void* hi, void* lo,
                           long long rows, int c, float eps, cudaStream_t stream) {
  if (rows == 0) return 0;
  if (c != 512) {
    set_error("layernorm_split is specialised for 512 channels (got %d)", c);
    return -2;
  }
  const int threads = 256, rows_per_block = 2 * (threads / 32);
  layernorm_split_kernel<16><<<static_cast<unsigned>((rows + rows_per_block - 1) / rows_per_block), threads, 0, stream>>>(
      x, gamma, beta, out, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), rows, eps);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
