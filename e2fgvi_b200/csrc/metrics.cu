// Per-frame PSNR and SSIM inputs of evaluate.py (reference core/metrics.py:20-54): the exact sum of squared errors
// and skimage 0.16.2's compare_ssim(data_range=R, multichannel=True, win_size=win), uniform window, sample covariance.
//
// One fused pass: a CTA owns kTile output columns of one frame (kTile + win - 1 input columns, the window's halo
// included) and walks down the rows.  Per input column it slides fp64 vertical sums of x, y, x^2, y^2 and xy over the
// last `win` rows (shared memory, each column updated by one thread).  Once `win` rows are in, every output row is a
// block-wide inclusive scan of those sums along the row, and an output's horizontal window sum is the difference of
// two scan values.  S is evaluated per output pixel and summed per thread; the SSE of the CTA's own columns is
// accumulated on the way.  Nothing but per-CTA partials goes to global memory, and a second kernel adds them per
// frame in a fixed order (no atomics: deterministic).
//
// Exactness: for uint8 operands or evaluate.py's composite (multiples of 1/4 in [0, 255]) every value added here is a
// multiple of 1/16, and every partial sum (column sums, row scans, SSE up to 1080p) is below 2^43, so all of them are
// exact in fp64 in any order.  The box means sum / win^2 are then correctly rounded (scipy's running uniform_filter1d
// is not), and S follows skimage's order of operations with explicit _rn intrinsics, so no FMA contraction changes a
// rounding.  Arbitrary fp32 operands get fp64 accumulation.
#include <cstdint>
#include "launch.h"

namespace e2f {
namespace metrics {

constexpr int kThreads = 256;   // one output column per thread
constexpr int kTile = kThreads;

struct Params {
  const void* a;
  const void* b;
  int a_u8, b_u8;
  int h, w, win, span, tiles;
  double npix, cov_norm, c1, c2;   // win^2, win^2 / (win^2 - 1), (0.01 R)^2, (0.03 R)^2
  double* work;                 // [n][tiles][1 + C]: SSE, then per-channel sums of S
};

__device__ __forceinline__ double load(const void* p, int u8, long long i) {
  return u8 ? static_cast<double>(static_cast<const uint8_t*>(p)[i]) : static_cast<double>(static_cast<const float*>(p)[i]);
}

// the five quantities of channel c sit at q = 5c + {x, y, xx, yy, xy}
template <int C>
__device__ __forceinline__ void add_row(const Params& p, long long base, double sign, double* v, bool own_sse,
                                        double& sse) {
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const double x = load(p.a, p.a_u8, base + c), y = load(p.b, p.b_u8, base + c);
    v[5 * c + 0] = __dadd_rn(v[5 * c + 0], sign * x);
    v[5 * c + 1] = __dadd_rn(v[5 * c + 1], sign * y);
    v[5 * c + 2] = __dadd_rn(v[5 * c + 2], sign * __dmul_rn(x, x));
    v[5 * c + 3] = __dadd_rn(v[5 * c + 3], sign * __dmul_rn(y, y));
    v[5 * c + 4] = __dadd_rn(v[5 * c + 4], sign * __dmul_rn(x, y));
    if (own_sse) {
      const double d = __dsub_rn(x, y);
      sse = __dadd_rn(sse, __dmul_rn(d, d));
    }
  }
}

// skimage 0.16.2 _structural_similarity.py, line for line, on the five window sums of one channel
__device__ __forceinline__ double ssim_of(const Params& p, const double* s) {
  const double ux = __ddiv_rn(s[0], p.npix), uy = __ddiv_rn(s[1], p.npix);
  const double uxx = __ddiv_rn(s[2], p.npix), uyy = __ddiv_rn(s[3], p.npix), uxy = __ddiv_rn(s[4], p.npix);
  const double vx = __dmul_rn(p.cov_norm, __dsub_rn(uxx, __dmul_rn(ux, ux)));
  const double vy = __dmul_rn(p.cov_norm, __dsub_rn(uyy, __dmul_rn(uy, uy)));
  const double vxy = __dmul_rn(p.cov_norm, __dsub_rn(uxy, __dmul_rn(ux, uy)));
  const double a1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), p.c1);
  const double a2 = __dadd_rn(__dmul_rn(2.0, vxy), p.c2);
  const double b1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), p.c1);
  const double b2 = __dadd_rn(__dadd_rn(vx, vy), p.c2);
  return __ddiv_rn(__dmul_rn(a1, a2), __dmul_rn(b1, b2));
}

// grid: n * tiles CTAs (frame-major).  Dynamic shared memory (all of the kernel's): vsum and scan, [5C][span] doubles
// each, then the per-warp scan totals, [kThreads / 32][5C].
template <int C>
__global__ void __launch_bounds__(kThreads, 1) frame_metrics_kernel(Params p) {
  constexpr int Q = 5 * C;
  extern __shared__ double smem[];
  double* vsum = smem;                          // [Q][span] sliding column sums
  double* scan = smem + Q * p.span;             // [Q][span] inclusive row scan of vsum
  double* warp_tot = scan + Q * p.span;         // [kThreads / 32][Q]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int frame = blockIdx.x / p.tiles, tile = blockIdx.x - frame * p.tiles;
  const int x0 = tile * kTile;
  const int span = p.span, win = p.win;
  const int wo = p.w - win + 1;
  const bool last = tile == p.tiles - 1;
  const long long frame_base = static_cast<long long>(frame) * p.h * p.w;

  for (int j = tid; j < Q * span; j += kThreads) vsum[j] = 0.0;
  double sse = 0.0, ssum[C];
#pragma unroll
  for (int c = 0; c < C; ++c) ssum[c] = 0.0;

  for (int y = 0; y < p.h; ++y) {
    // vertical slide: add row y, drop row y - win.  Column j is only ever touched by thread j % kThreads, here and
    // in the scan's load below, so no barrier separates the two.
    for (int j = tid; j < span && x0 + j < p.w; j += kThreads) {
      double v[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) v[q] = vsum[q * span + j];
      const bool own = j < kTile || last;      // the CTA's own columns, for the SSE
      add_row<C>(p, (frame_base + static_cast<long long>(y) * p.w + x0 + j) * C, 1.0, v, own, sse);
      if (y >= win) add_row<C>(p, (frame_base + static_cast<long long>(y - win) * p.w + x0 + j) * C, -1.0, v, false, sse);
#pragma unroll
      for (int q = 0; q < Q; ++q) vsum[q * span + j] = v[q];
    }
    if (y < win - 1) continue;

    // inclusive scan of vsum along the row, kThreads columns at a time with a running carry
    double carry[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) carry[q] = 0.0;
    for (int k = 0; k < span; k += kThreads) {
      const int j = k + tid;
      double v[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) v[q] = j < span ? vsum[q * span + j] : 0.0;   // zero past the frame's edge
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
#pragma unroll
        for (int q = 0; q < Q; ++q) {
          const double t = __shfl_up_sync(0xffffffffu, v[q], off);
          if (lane >= off) v[q] = __dadd_rn(v[q], t);
        }
      }
      if (lane == 31) {
#pragma unroll
        for (int q = 0; q < Q; ++q) warp_tot[warp * Q + q] = v[q];
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        double run = carry[q], mine = 0.0;     // carry + totals of the warps before this one
        for (int u = 0; u < kThreads / 32; ++u) {
          if (u == warp) mine = run;
          run = __dadd_rn(run, warp_tot[u * Q + q]);
        }
        carry[q] = run;
        if (j < span) scan[q * span + j] = __dadd_rn(v[q], mine);
      }
      __syncthreads();
    }

    // output row y - win + 1, column x0 + tid: window sums = scan[tid + win - 1] - scan[tid - 1]
    if (x0 + tid < wo) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        double s[5];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          const int q = 5 * c + i;
          const double hi = scan[q * span + tid + win - 1];
          s[i] = tid ? __dsub_rn(hi, scan[q * span + tid - 1]) : hi;
        }
        ssum[c] = __dadd_rn(ssum[c], ssim_of(p, s));
      }
    }
    __syncthreads();    // the next row's scan overwrites `scan`
  }

  // fixed-order block reduction of (sse, ssum[C]) into this CTA's partials
  double* red = smem;   // reuses vsum: kThreads * (1 + C) doubles <= Q * span
  red[tid] = sse;
#pragma unroll
  for (int c = 0; c < C; ++c) red[(1 + c) * kThreads + tid] = ssum[c];
  __syncthreads();
  for (int stride = kThreads / 2; stride > 0; stride >>= 1) {
    if (tid < stride)
      for (int i = 0; i <= C; ++i) red[i * kThreads + tid] = __dadd_rn(red[i * kThreads + tid], red[i * kThreads + tid + stride]);
    __syncthreads();
  }
  if (tid <= C) p.work[static_cast<long long>(blockIdx.x) * (1 + C) + tid] = red[tid * kThreads];
}

// SSE only (win = 0): a CTA sums kSseElems consecutive values of one frame; grid n * blocks, frame-major
constexpr int kSseElems = kThreads * 16;

__global__ void __launch_bounds__(kThreads) frame_sse_kernel(const void* __restrict__ a, int a_u8,
                                                             const void* __restrict__ b, int b_u8, long long elems,
                                                             int blocks, double* __restrict__ work) {
  __shared__ double red[kThreads];
  const int tid = threadIdx.x;
  const int frame = blockIdx.x / blocks, blk = blockIdx.x - frame * blocks;
  const long long base = static_cast<long long>(frame) * elems, lo = static_cast<long long>(blk) * kSseElems;
  const long long hi = lo + kSseElems < elems ? lo + kSseElems : elems;
  double s = 0.0;
  for (long long i = lo + tid; i < hi; i += kThreads) {
    const double d = __dsub_rn(load(a, a_u8, base + i), load(b, b_u8, base + i));
    s = __dadd_rn(s, __dmul_rn(d, d));
  }
  red[tid] = s;
  __syncthreads();
  for (int stride = kThreads / 2; stride > 0; stride >>= 1) {
    if (tid < stride) red[tid] = __dadd_rn(red[tid], red[tid + stride]);
    __syncthreads();
  }
  if (tid == 0) work[blockIdx.x] = red[0];
}

// one thread per frame: tiles in order; SSIM = mean over channels of (sum of S) / (ho * wo), when ssim is given
__global__ void frame_metrics_reduce_kernel(const double* __restrict__ work, double* __restrict__ sse,
                                            double* __restrict__ ssim, int n, int tiles, int c, double count) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const double* w = work + static_cast<long long>(f) * tiles * (1 + c);
  double e = 0.0;
  for (int t = 0; t < tiles; ++t) e = __dadd_rn(e, w[t * (1 + c)]);
  double m = 0.0;
  for (int ch = 0; ch < c; ++ch) {
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s = __dadd_rn(s, w[t * (1 + c) + 1 + ch]);
    m = __dadd_rn(m, __ddiv_rn(s, count));
  }
  sse[f] = e;
  if (ssim) ssim[f] = __ddiv_rn(m, static_cast<double>(c));
}

}  // namespace metrics

int frame_metrics_tiles(int w, int win) { return (w - win + 1 + metrics::kTile - 1) / metrics::kTile; }

long long frame_sse_blocks(int h, int w, int c) {
  return (static_cast<long long>(h) * w * c + metrics::kSseElems - 1) / metrics::kSseElems;
}

size_t frame_metrics_smem(int c, int win) {
  return sizeof(double) * 5 * static_cast<size_t>(c) * (2 * (metrics::kTile + win - 1) + metrics::kThreads / 32);
}

int launch_frame_sse(const void* a, int a_u8, const void* b, int b_u8, double* sse, double* work, int n, int h, int w,
                     int c, cudaStream_t stream) {
  const long long elems = static_cast<long long>(h) * w * c;
  const int blocks = static_cast<int>(frame_sse_blocks(h, w, c));
  metrics::frame_sse_kernel<<<static_cast<unsigned>(static_cast<long long>(n) * blocks), metrics::kThreads, 0, stream>>>(
      a, a_u8, b, b_u8, elems, blocks, work);
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  metrics::frame_metrics_reduce_kernel<<<(n + 127) / 128, 128, 0, stream>>>(work, sse, nullptr, n, blocks, 0, 1.0);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_frame_metrics(const void* a, int a_u8, const void* b, int b_u8, double* sse, double* ssim, double* work,
                         int n, int h, int w, int c, int win, double data_range, cudaStream_t stream) {
  metrics::Params p;
  p.a = a; p.b = b; p.a_u8 = a_u8; p.b_u8 = b_u8;
  p.h = h; p.w = w; p.win = win;
  p.span = metrics::kTile + win - 1;
  p.tiles = frame_metrics_tiles(w, win);
  const long long np_ = static_cast<long long>(win) * win;
  p.npix = static_cast<double>(np_);
  p.cov_norm = static_cast<double>(np_) / static_cast<double>(np_ - 1);
  p.c1 = (0.01 * data_range) * (0.01 * data_range);
  p.c2 = (0.03 * data_range) * (0.03 * data_range);
  p.work = work;
  const size_t smem = frame_metrics_smem(c, win);
  const unsigned grid = static_cast<unsigned>(static_cast<long long>(n) * p.tiles);
  cudaError_t e = cudaSuccess;
  switch (c) {
#define E2F_METRICS_CASE(C)                                                                                        \
    case C:                                                                                                          \
      e = cudaFuncSetAttribute(metrics::frame_metrics_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,        \
                               static_cast<int>(smem));                                                              \
      if (e != cudaSuccess) return static_cast<int>(e);                                                              \
      metrics::frame_metrics_kernel<C><<<grid, metrics::kThreads, smem, stream>>>(p);                                \
      break;
    E2F_METRICS_CASE(1)
    E2F_METRICS_CASE(2)
    E2F_METRICS_CASE(3)
    E2F_METRICS_CASE(4)
#undef E2F_METRICS_CASE
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  count_launch();
  e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  const double count = static_cast<double>(h - win + 1) * static_cast<double>(w - win + 1);
  metrics::frame_metrics_reduce_kernel<<<(n + 127) / 128, 128, 0, stream>>>(work, sse, ssim, n, p.tiles, c, count);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
