// Backward of the transformer blocks' LayerNorms and focal window pooling (the adjoints of elementwise.cu's
// layernorm_split_kernel and layernorm_pool_split_kernel), C = 512:
//   layernorm_backward      : dx = residual + rstd * (g - mean(g) - x^ * mean(g * x^)), g = gamma * dy, x^ = (x - mean) *
//                             rstd, recomputed from the kept fp32 x in the forward's two-pass order; fp32 and/or split out
//   layernorm_pool_backward : the same with dy = dxn + w_pool[token] * dpooled[window], one CTA per (frame, window), and
//                             d w_pool[token] = sum_c dpooled * LN(x)[token], d b_pool = sum_c dpooled
// The parameter gradients leave each CTA as one partial row and column_sum_kernel adds the rows in a fixed order: no
// atomics, bit-identical from run to run.  HBM-bound; algorithmic bytes = inputs read + outputs written.
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace {

constexpr int LN_C = 512, LN_PER_LANE = LN_C / 32, LN_WARPS = 8;
constexpr int LN_PAIRS_PER_WARP = 4;
constexpr int LN_ROWS_PER_CTA = LN_WARPS * LN_PAIRS_PER_WARP * 2;     // 64 rows: one partial row per 64 input rows

__device__ __forceinline__ void load_row(const float* __restrict__ r, int lane, float (&v)[LN_PER_LANE]) {
#pragma unroll
  for (int j = 0; j < LN_PER_LANE / 8; ++j) {       // lane owns 8 consecutive floats per 256-float segment (as the forward)
    const float4 a = __ldg(reinterpret_cast<const float4*>(r + j * 256 + lane * 8));
    const float4 b = __ldg(reinterpret_cast<const float4*>(r + j * 256 + lane * 8) + 1);
    v[8 * j + 0] = a.x; v[8 * j + 1] = a.y; v[8 * j + 2] = a.z; v[8 * j + 3] = a.w;
    v[8 * j + 4] = b.x; v[8 * j + 5] = b.y; v[8 * j + 6] = b.z; v[8 * j + 7] = b.w;
  }
}

__device__ __forceinline__ void load_params(const float* __restrict__ p, int lane, float (&v)[LN_PER_LANE]) {
#pragma unroll
  for (int j = 0; j < LN_PER_LANE / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[8 * j + e] = __ldg(p + j * 256 + lane * 8 + e);
  }
}

__device__ __forceinline__ float warp_sum(float s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// mean and rstd exactly as layernorm_split_kernel / layernorm_pool_split_kernel compute them
__device__ __forceinline__ void row_stats(const float (&v)[LN_PER_LANE], float eps, float& mean, float& rstd) {
  float sum = 0.f;
#pragma unroll
  for (int e = 0; e < LN_PER_LANE; ++e) sum += v[e];
  mean = warp_sum(sum) * (1.0f / LN_C);
  float sq = 0.f;
#pragma unroll
  for (int e = 0; e < LN_PER_LANE; ++e) {
    const float d = v[e] - mean;
    sq = fmaf(d, d, sq);
  }
  rstd = rsqrtf(warp_sum(sq) * (1.0f / LN_C) + eps);
}

// The input gradient of one row, in place of dy: dy <- rstd * (g - mean(g) - x^ mean(g x^)) with g = gamma * dy;
// v <- x^.  Accumulates dy * x^ and dy into the parameter sums when `acc`.
__device__ __forceinline__ void row_backward(float (&v)[LN_PER_LANE], float (&d)[LN_PER_LANE],
                                             const float (&gm)[LN_PER_LANE], float mean, float rstd, bool acc,
                                             float (&ag)[LN_PER_LANE], float (&ab)[LN_PER_LANE]) {
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int e = 0; e < LN_PER_LANE; ++e) {
    v[e] = (v[e] - mean) * rstd;
    if (acc) {
      ag[e] = fmaf(d[e], v[e], ag[e]);
      ab[e] += d[e];
    }
    d[e] *= gm[e];
    s1 += d[e];
    s2 = fmaf(d[e], v[e], s2);
  }
  const float m1 = warp_sum(s1) * (1.0f / LN_C), m2 = warp_sum(s2) * (1.0f / LN_C);
#pragma unroll
  for (int e = 0; e < LN_PER_LANE; ++e) d[e] = rstd * (d[e] - m1 - v[e] * m2);
}

__device__ __forceinline__ void split_store8(const float* f, __nv_bfloat16* hi, __nv_bfloat16* lo) {
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

// out (+ residual) of one row: fp32 and/or the bf16 (hi, lo) split
__device__ __forceinline__ void store_row(float (&d)[LN_PER_LANE], const float* __restrict__ res, float* __restrict__ out,
                                          __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long row,
                                          int lane) {
  if (res) {
    float r[LN_PER_LANE];
    load_row(res + row * LN_C, lane, r);
#pragma unroll
    for (int e = 0; e < LN_PER_LANE; ++e) d[e] += r[e];
  }
#pragma unroll
  for (int j = 0; j < LN_PER_LANE / 8; ++j) {
    const long long o = row * LN_C + j * 256 + lane * 8;
    if (out) {
      float4* d4 = reinterpret_cast<float4*>(out + o);
      d4[0] = make_float4(d[8 * j + 0], d[8 * j + 1], d[8 * j + 2], d[8 * j + 3]);
      d4[1] = make_float4(d[8 * j + 4], d[8 * j + 5], d[8 * j + 6], d[8 * j + 7]);
    }
    if (hi) split_store8(&d[8 * j], hi + o, lo + o);
  }
}

// The 8 warps' (dgamma | dbeta) sums added in warp order through shared memory, written as the CTA's partial row.
__device__ __forceinline__ void store_param_partials(float (*red)[2 * LN_C], const float (&ag)[LN_PER_LANE],
                                                     const float (&ab)[LN_PER_LANE], float* __restrict__ prow, int warp,
                                                     int lane) {
#pragma unroll
  for (int j = 0; j < LN_PER_LANE / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      red[warp][j * 256 + lane * 8 + e] = ag[8 * j + e];
      red[warp][LN_C + j * 256 + lane * 8 + e] = ab[8 * j + e];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * LN_C; c += blockDim.x) {
    float t = red[0][c];
#pragma unroll
    for (int k = 1; k < LN_WARPS; ++k) t += red[k][c];
    prow[c] = t;
  }
}

// One warp per pair of rows (both rows' loads in flight before the first reduction, as the forward), 4 pairs per warp,
// 64 rows per CTA; an odd last row is handled alone.
__global__ void __launch_bounds__(256) layernorm_backward_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ res, float* __restrict__ out,
                                                                 __nv_bfloat16* __restrict__ hi,
                                                                 __nv_bfloat16* __restrict__ lo,
                                                                 float* __restrict__ part, long long rows, float eps) {
  constexpr int R = 2;
  __shared__ float red[LN_WARPS][2 * LN_C];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool acc = part != nullptr, write = out != nullptr || hi != nullptr;
  float gm[LN_PER_LANE], ag[LN_PER_LANE], ab[LN_PER_LANE];
  load_params(gamma, lane, gm);
#pragma unroll
  for (int e = 0; e < LN_PER_LANE; ++e) ag[e] = ab[e] = 0.f;
  const long long base = static_cast<long long>(blockIdx.x) * LN_ROWS_PER_CTA;
  for (int it = 0; it < LN_PAIRS_PER_WARP; ++it) {
    const long long row0 = base + (it * LN_WARPS + warp) * R;
    if (row0 >= rows) break;
    float v[R][LN_PER_LANE], d[R][LN_PER_LANE];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long long row = row0 + (row0 + r < rows ? r : 0);
      load_row(x + row * LN_C, lane, v[r]);
      load_row(dy + row * LN_C, lane, d[r]);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (row0 + r >= rows) break;
      float mean, rstd;
      row_stats(v[r], eps, mean, rstd);
      row_backward(v[r], d[r], gm, mean, rstd, acc, ag, ab);
      if (write) store_row(d[r], res, out, hi, lo, row0 + r, lane);
    }
  }
  if (acc) store_param_partials(red, ag, ab, part + static_cast<long long>(blockIdx.x) * 2 * LN_C, warp, lane);
}

// One CTA per (frame, window), each warp whole token rows (the forward's assignment).  Partial row of the CTA:
// [dgamma (512) | dbeta (512) | d w_pool (wh*ww) | d b_pool (1)].
__global__ void __launch_bounds__(256) layernorm_pool_backward_kernel(
    const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
    const float* __restrict__ pool_w, const float* __restrict__ drows, const float* __restrict__ dx1,
    float* __restrict__ out, float* __restrict__ part, int H, int W, int wh, int ww, long long n_tok, int want_norm,
    int want_pool, float eps) {
  __shared__ float red[LN_WARPS][2 * LN_C];
  const int nww = W / ww, nwh = H / wh, ntok = wh * ww;
  const int win = blockIdx.x, bt = blockIdx.y;
  const int wi = win / nww, wj = win - wi * nww;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long cta = static_cast<long long>(bt) * nwh * nww + win;
  float* prow = part ? part + cta * (2 * LN_C + ntok + 1) : nullptr;
  float gm[LN_PER_LANE], bt_[LN_PER_LANE], dp[LN_PER_LANE], ag[LN_PER_LANE], ab[LN_PER_LANE];
  load_params(gamma, lane, gm);
  load_params(beta, lane, bt_);
  load_row(drows + (n_tok + cta) * LN_C, lane, dp);            // dpooled of this window: pooled rows follow the tokens
#pragma unroll
  for (int e = 0; e < LN_PER_LANE; ++e) ag[e] = ab[e] = 0.f;
  if (want_pool && warp == 0) {
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < LN_PER_LANE; ++e) s += dp[e];
    s = warp_sum(s);
    if (lane == 0) prow[2 * LN_C + ntok] = s;
  }
  for (int tok = warp; tok < ntok; tok += LN_WARPS) {
    const int r = tok / ww, q = tok - r * ww;
    const long long row = (static_cast<long long>(bt) * H + wi * wh + r) * W + wj * ww + q;
    float v[LN_PER_LANE], d[LN_PER_LANE];
    load_row(x + row * LN_C, lane, v);
    load_row(drows + row * LN_C, lane, d);
    const float wt = __ldg(pool_w + tok);
    float mean, rstd;
    row_stats(v, eps, mean, rstd);
    if (want_pool) {                                 // d w_pool[tok] = sum_c dpooled * LN(x) at the fp32 affine output
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < LN_PER_LANE; ++e) s = fmaf(dp[e], (v[e] - mean) * rstd * gm[e] + bt_[e], s);
      s = warp_sum(s);
      if (lane == 0) prow[2 * LN_C + tok] = s;
    }
#pragma unroll
    for (int e = 0; e < LN_PER_LANE; ++e) d[e] = fmaf(wt, dp[e], d[e]);
    row_backward(v, d, gm, mean, rstd, want_norm != 0, ag, ab);
    if (out) store_row(d, dx1, out, nullptr, nullptr, row, lane);
  }
  if (want_norm) store_param_partials(red, ag, ab, prow, warp, lane);
}

// Sinks of the fixed-order column sum: columns [end[s-1], end[s]) of the partial rows go to dst[s] (NULL: not wanted).
struct ColumnSinks {
  float* dst[4];
  int end[4];
};

// sums[c] = sum over the partial rows p = 0 .. nparts-1 of part[p][c] for c in [col0, col1): 8 row groups of 32 columns
// per CTA, each group adds rows g, g + 8, ... in order, then the 8 group sums are added in group order.
__global__ void __launch_bounds__(256) column_sum_kernel(const float* __restrict__ part, int nparts, int ld, int col0,
                                                         int col1, ColumnSinks sinks) {
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int col = col0 + blockIdx.x * 32 + lane;
  float s = 0.f;
  if (col < col1) {
    for (int p = grp; p < nparts; p += 8) s += __ldg(part + static_cast<long long>(p) * ld + col);
  }
  red[grp][lane] = s;
  __syncthreads();
  if (grp != 0 || col >= col1) return;
  float t = red[0][lane];
#pragma unroll
  for (int k = 1; k < 8; ++k) t += red[k][lane];
  // (a chain of selects, not an indexed load: the sinks stay in parameter space)
  float* dst = sinks.dst[0];
  int start = 0;
#pragma unroll
  for (int s = 1; s < 4; ++s) {
    if (col >= sinks.end[s - 1]) {
      dst = sinks.dst[s];
      start = sinks.end[s - 1];
    }
  }
  if (dst) dst[col - start] = t;
}

int launch_column_sum(const float* part, int nparts, int ld, int col0, int col1, const ColumnSinks& sinks,
                      cudaStream_t stream) {
  column_sum_kernel<<<(col1 - col0 + 31) / 32, 256, 0, stream>>>(part, nparts, ld, col0, col1, sinks);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace

long long layernorm_backward_parts(long long rows) { return (rows + LN_ROWS_PER_CTA - 1) / LN_ROWS_PER_CTA; }

long long layernorm_backward_work_elems(long long rows) { return layernorm_backward_parts(rows) * 2 * LN_C; }

long long layernorm_pool_backward_work_elems(int bt, int h, int w, int wh, int ww) {
  return static_cast<long long>(bt) * (h / wh) * (w / ww) * (2 * LN_C + wh * ww + 1);
}

int launch_layernorm_backward(const float* x, const float* dy, const float* gamma, const float* res, float* out, void* hi,
                              void* lo, float* dgamma, float* dbeta, float* work, long long rows, int c, float eps,
                              cudaStream_t stream) {
  if (c != LN_C) {
    set_error("layernorm_backward is specialised for 512 channels (got %d)", c);
    return -2;
  }
  if (rows == 0) {
    if (dgamma) cudaMemsetAsync(dgamma, 0, LN_C * sizeof(float), stream);
    if (dbeta) cudaMemsetAsync(dbeta, 0, LN_C * sizeof(float), stream);
    return static_cast<int>(cudaGetLastError());
  }
  const long long parts = layernorm_backward_parts(rows);
  if (parts > 0x7fffffffLL) {
    set_error("layernorm_backward: %lld rows is too many for one launch", rows);
    return -2;
  }
  float* part = (dgamma || dbeta) ? work : nullptr;
  layernorm_backward_kernel<<<static_cast<unsigned>(parts), 256, 0, stream>>>(
      x, dy, gamma, res, out, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), part, rows, eps);
  count_launch();
  int st = static_cast<int>(cudaGetLastError());
  if (st || !part) return st;
  const ColumnSinks sinks{{dgamma, dbeta, nullptr, nullptr}, {LN_C, 2 * LN_C, 2 * LN_C, 2 * LN_C}};
  return launch_column_sum(part, static_cast<int>(parts), 2 * LN_C, dgamma ? 0 : LN_C, dbeta ? 2 * LN_C : LN_C, sinks,
                           stream);
}

int launch_layernorm_pool_backward(const float* x, const float* gamma, const float* beta, const float* pool_w,
                                   const float* drows, const float* dx1, float* out, float* dgamma, float* dbeta,
                                   float* dpool_w, float* dpool_b, float* work, int bt, int h, int w, int c, int wh,
                                   int ww, float eps, cudaStream_t stream) {
  if (c != LN_C) {
    set_error("layernorm_pool_backward is specialised for 512 channels (got %d)", c);
    return -2;
  }
  const int ntok = wh * ww, ld = 2 * LN_C + ntok + 1;
  const bool want_norm = dgamma || dbeta, want_pool = dpool_w || dpool_b;
  if (bt == 0) {
    if (dgamma) cudaMemsetAsync(dgamma, 0, LN_C * sizeof(float), stream);
    if (dbeta) cudaMemsetAsync(dbeta, 0, LN_C * sizeof(float), stream);
    if (dpool_w) cudaMemsetAsync(dpool_w, 0, ntok * sizeof(float), stream);
    if (dpool_b) cudaMemsetAsync(dpool_b, 0, sizeof(float), stream);
    return static_cast<int>(cudaGetLastError());
  }
  const dim3 grid((h / wh) * (w / ww), bt);
  float* part = (want_norm || want_pool) ? work : nullptr;
  layernorm_pool_backward_kernel<<<grid, 256, 0, stream>>>(x, gamma, beta, pool_w, drows, dx1, out, part, h, w, wh, ww,
                                                           static_cast<long long>(bt) * h * w, want_norm ? 1 : 0,
                                                           want_pool ? 1 : 0, eps);
  count_launch();
  int st = static_cast<int>(cudaGetLastError());
  if (st || !part) return st;
  const ColumnSinks sinks{{dgamma, dbeta, dpool_w, dpool_b}, {LN_C, 2 * LN_C, 2 * LN_C + ntok, ld}};
  const int col0 = want_norm ? (dgamma ? 0 : LN_C) : 2 * LN_C;
  const int col1 = want_pool ? (dpool_b ? ld : ld - 1) : (dbeta ? 2 * LN_C : LN_C);
  return launch_column_sum(part, static_cast<int>(grid.x * grid.y), ld, col0, col1, sinks, stream);
}

}  // namespace e2f
