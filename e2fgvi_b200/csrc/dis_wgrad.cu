// Weight and bias gradients of the discriminator's Conv3d layers (kernel 3x5x5, stride (1, 2, 2), padding
// (1, pad, pad)), see launch_dis_conv for the forward:
//     dW[co][ci][kt][ky][kx] = sum over (b, t, y, x) of dY[b][t][y][x][co] * X[b][t + kt - 1][2y + ky - pad][2x + kx - pad][ci]
//     db[co]                 = sum over (b, t, y, x) of dY[b][t][y][x][co]
// and of SPyNet's 2-D 7x7 / stride 1 / pad 3 convs (KT = 1, KS = 7, S = 1), whose X is dense or row-gapped (each image
// row `x_lead` zero pixels in front, `x_pitch` pixels apart: the operand the forward conv read).
// dW is a GEMM with M = cout, N = TAPS * cin (column j = tap * cin + ci, taps in (kt, ky, kx) order) and K = the output
// pixels, on wgmma with the bf16 three-term split and fp32 accumulation (the accuracy class of the forward convs).
//  * One warpgroup per CTA computes a 64 (co) x 128 (j) tile over one K slice, 64 pixels per K block.  Both operands
//    are pixel-major in memory and the B operand is a gather (each column group reads its own tap's shifted, strided,
//    zero-padded pixels), so the warpgroup stages them itself into the K-major 128-byte-swizzled layout the wgmma
//    descriptors read: dY is split into (hi, lo) as it is loaded, X's (hi, lo) come 8 channels per 16-byte load.
//    Two stage buffers: the loads of block i + 1 overlap the MMAs of block i.
//  * K is split into `slices` contiguous pixel ranges, one per blockIdx.z; each writes its partial tile to the fp32
//    workspace and a second kernel adds the slices in slice order, so the result is bit-identical from run to run (no
//    atomics).
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace wgrad {

constexpr int MT = 64, NT = 128, KB = 64, THREADS = 128;
constexpr int A_PART = MT * 128, B_PART = NT * 128;          // one bf16 part (hi or lo) of a K block, 128-byte rows
constexpr int BUF = 2 * A_PART + 2 * B_PART;                 // [Ah | Al | Bh | Bl] = 48 KB
constexpr int SMEM = 2 * BUF + 1024;

// Pixel ranges are whole K blocks; the slice count depends on the shape alone.
__host__ __device__ inline long long slice_len(long long pixels, int slices) {
  const long long per = (pixels + slices - 1) / slices;
  return (per + KB - 1) / KB * KB;
}

__device__ __forceinline__ uint32_t pack_bf2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}

// element pair (k, k + 1), k even, of row `row` in a K-major SW128 tile
__device__ __forceinline__ void st_pair(uint32_t base, int row, int k, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(base + sw128_offset(row, k >> 3) + (k & 7) * 2), "r"(v) : "memory");
}

// Tap (kt, ky, kx) of output pixel (t, y, x) reads X at (t + kt - KT / 2, S y + ky - pad, S x + kx - pad).
template <int KT, int KS, int S>
__global__ void __launch_bounds__(THREADS) wgrad_mma_kernel(const float* __restrict__ dy, const __nv_bfloat16* __restrict__ xh,
                                                            const __nv_bfloat16* __restrict__ xl, float* __restrict__ ws,
                                                            int b, int t, int h_in, int w_in, int x_pitch, int x_lead,
                                                            int cin, int h_o, int w_o, int cout, int pad, int slices) {
  constexpr int TAPS = KT * KS * KS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * MT, n0 = blockIdx.x * NT;
  const int N = TAPS * cin;
  const long long pixels = static_cast<long long>(b) * t * h_o * w_o;
  const long long len = slice_len(pixels, slices);
  const long long k0 = len * blockIdx.z;
  const long long k1 = k0 + len < pixels ? k0 + len : pixels;
  // B staging tasks of this thread: (pixel pair kp, column group jg of 8 channels of one tap), q = tid + 128 r
  int bdt[4], bdy[4], bdx[4], bci[4];
  bool bok[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int j0 = n0 + 8 * ((tid + THREADS * r) >> 5);
    bok[r] = j0 < N;
    const int tap = bok[r] ? j0 / cin : 0;
    bci[r] = bok[r] ? j0 - tap * cin : 0;
    bdt[r] = tap / (KS * KS) - KT / 2;
    bdy[r] = (tap / KS) % KS - pad;
    bdx[r] = tap % KS - pad;
  }
  float acc[NT / 2];                                    // overwritten by the first MMA (scale-d = 0)
  const uint32_t s0 = smem_u32(smem);
  int it = 0;
  for (long long base = k0; base < k1; base += KB, ++it) {
    const uint32_t buf = s0 + (it & 1) * BUF;
    const uint32_t a_hi = buf, a_lo = buf + A_PART, b_hi = buf + 2 * A_PART, b_lo = b_hi + B_PART;
    // ---- A = dY^T: rows co, K = pixels; task (kp, co group cg), q = tid + 128 r
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = tid + THREADS * r, kp = q & 31, cg = q >> 5;
      const int co = m0 + 8 * cg;
      float v[2][8];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const long long k = base + 2 * kp + e;
        if (k < k1 && co < cout) {
          const float4* src = reinterpret_cast<const float4*>(dy + k * cout + co);
          const float4 p0 = __ldg(src), p1 = __ldg(src + 1);
          v[e][0] = p0.x; v[e][1] = p0.y; v[e][2] = p0.z; v[e][3] = p0.w;
          v[e][4] = p1.x; v[e][5] = p1.y; v[e][6] = p1.z; v[e][7] = p1.w;
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) v[e][c] = 0.f;
        }
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(v[0][c]), h1 = __float2bfloat16_rn(v[1][c]);
        const __nv_bfloat16 l0 = __float2bfloat16_rn(v[0][c] - __bfloat162float(h0));
        const __nv_bfloat16 l1 = __float2bfloat16_rn(v[1][c] - __bfloat162float(h1));
        st_pair(a_hi, 8 * cg + c, 2 * kp, pack_bf2(h0, h1));
        st_pair(a_lo, 8 * cg + c, 2 * kp, pack_bf2(l0, l1));
      }
    }
    // ---- B = gathered X: rows j = (tap, ci), K = pixels; task (kp, column group jg)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int q = tid + THREADS * r, kp = q & 31, jg = q >> 5;
      uint4 vh[2], vl[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        vh[e] = vl[e] = make_uint4(0, 0, 0, 0);
        const long long k = base + 2 * kp + e;
        if (bok[r] && k < k1) {
          const int x = static_cast<int>(k % w_o);
          const long long rr = k / w_o;
          const int y = static_cast<int>(rr % h_o);
          const long long n = rr / h_o;                        // b * t + frame
          const int fr = static_cast<int>(n % t);
          const int ti = fr + bdt[r], yi = S * y + bdy[r], xi = S * x + bdx[r];
          if (ti >= 0 && ti < t && yi >= 0 && yi < h_in && xi >= 0 && xi < w_in) {
            const long long off = (((n + bdt[r]) * h_in + yi) * static_cast<long long>(x_pitch) + x_lead + xi) * cin + bci[r];
            vh[e] = __ldg(reinterpret_cast<const uint4*>(xh + off));
            vl[e] = __ldg(reinterpret_cast<const uint4*>(xl + off));
          }
        }
      }
      const __nv_bfloat16* h0 = reinterpret_cast<const __nv_bfloat16*>(&vh[0]);
      const __nv_bfloat16* h1 = reinterpret_cast<const __nv_bfloat16*>(&vh[1]);
      const __nv_bfloat16* l0 = reinterpret_cast<const __nv_bfloat16*>(&vl[0]);
      const __nv_bfloat16* l1 = reinterpret_cast<const __nv_bfloat16*>(&vl[1]);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        st_pair(b_hi, 8 * jg + c, 2 * kp, pack_bf2(h0[c], h1[c]));
        st_pair(b_lo, 8 * jg + c, 2 * kp, pack_bf2(l0[c], l1[c]));
      }
    }
    fence_proxy_async_smem();                           // generic-proxy stores -> wgmma operand reads
    __syncthreads();
    const uint64_t dah = gmma_desc_sw128(a_hi, 16, 1024), dal = gmma_desc_sw128(a_lo, 16, 1024);
    const uint64_t dbh = gmma_desc_sw128(b_hi, 16, 1024), dbl = gmma_desc_sw128(b_lo, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KB / 16; ++k) {
      wgmma_ss<NT, false>(acc, dal + 2 * k, dbh + 2 * k, (it | k) != 0);   // small terms first
      wgmma_ss<NT, false>(acc, dah + 2 * k, dbl + 2 * k, 1);
      wgmma_ss<NT, false>(acc, dah + 2 * k, dbh + 2 * k, 1);
    }
    wgmma_commit();
    wgmma_wait<1>();                                    // block it - 1 is done: its buffer is staged next
    __syncthreads();
  }
  wgmma_wait<0>();
  float* dst = ws + static_cast<size_t>(blockIdx.z) * cout * N;
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) {
    const int m = m0 + 16 * warp + (lane >> 2) + ((i >> 1) & 1) * 8;
    const int n = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    if (m < cout && n < N) dst[static_cast<size_t>(m) * N + n] = it ? acc[i] : 0.f;   // it == 0: an empty slice
  }
}

// Per-slice partial bias gradient: block z sums dY over its pixel range, thread = output channel.
__global__ void __launch_bounds__(128) bias_partial_kernel(const float* __restrict__ dy, float* __restrict__ ws, long long pixels,
                                                           int cout, int slices) {
  const long long len = slice_len(pixels, slices);
  const long long k0 = len * blockIdx.x;
  const long long k1 = k0 + len < pixels ? k0 + len : pixels;
  for (int co = threadIdx.x; co < cout; co += blockDim.x) {
    float s = 0.f;
    for (long long k = k0; k < k1; ++k) s += __ldg(dy + k * cout + co);
    ws[static_cast<size_t>(blockIdx.x) * cout + co] = s;
  }
}

// The same partials with the slice's pixels spread over the block: thread = (channel co, row r) for cout <= 128 (rows =
// 256 / cout threads per channel, consecutive threads read consecutive channels of one pixel), each thread sums pixels
// r, r + rows, ... of the slice (8 independent partial sums), and the rows are added in a fixed order.  Deterministic, and not latency-bound on a
// single thread per channel.
__global__ void __launch_bounds__(256) bias_partial_rows_kernel(const float* __restrict__ dy, float* __restrict__ ws,
                                                                long long pixels, int cout, int slices) {
  __shared__ float part[256];
  const long long len = slice_len(pixels, slices);
  const long long k0 = len * blockIdx.x;
  const long long k1 = k0 + len < pixels ? k0 + len : pixels;
  const int rows = 256 / cout, co = threadIdx.x % cout, r = threadIdx.x / cout;
  // eight independent sums per thread keep eight loads in flight; they are added in a fixed order
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (r < rows) {
    long long k = k0 + r;
    for (; k + 7 * rows < k1; k += 8 * rows) {
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] += __ldg(dy + (k + u * rows) * cout + co);
    }
    for (int u = 0; k < k1; k += rows, ++u) a[u] += __ldg(dy + k * cout + co);
  }
  part[threadIdx.x] = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]));
  __syncthreads();
  if (threadIdx.x < cout) {
    float t = 0.f;
    for (int i = 0; i < rows; ++i) t += part[i * cout + threadIdx.x];
    ws[static_cast<size_t>(blockIdx.x) * cout + threadIdx.x] = t;
  }
}

// dW[co][ci][tap] = sum over slices, in slice order, of ws[slice][co][tap * cin + ci]; the bias partials likewise.
template <int TAPS>
__global__ void __launch_bounds__(256) reduce_kernel(const float* __restrict__ ws, const float* __restrict__ wsb, float* __restrict__ dw,
                                                     float* __restrict__ db, int cout, int cin, int slices) {
  const int N = TAPS * cin;
  const long long total = static_cast<long long>(cout) * N;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) {
    const int m = static_cast<int>(i / N), j = static_cast<int>(i - static_cast<long long>(m) * N);
    float s = 0.f;
    for (int z = 0; z < slices; ++z) s += ws[static_cast<size_t>(z) * total + i];
    const int tap = j / cin, ci = j - tap * cin;
    dw[(static_cast<size_t>(m) * cin + ci) * TAPS + tap] = s;
  }
  if (db && i < cout) {
    float s = 0.f;
    for (int z = 0; z < slices; ++z) s += wsb[static_cast<size_t>(z) * cout + i];
    db[i] = s;
  }
}

}  // namespace wgrad

// Split-K slice count: enough CTAs to fill the GPU about twice at the tile count, at least 4 K blocks per slice, at
// most 64 slices.  A function of the shape alone, so results do not depend on the device.
static int wgrad_slices(long long pixels, int cout, int n_cols) {
  using namespace wgrad;
  const long long tiles = static_cast<long long>((cout + MT - 1) / MT) * ((n_cols + NT - 1) / NT);
  long long s = (264 + tiles - 1) / tiles;
  const long long cap = pixels / (4 * KB);
  if (s > cap) s = cap;
  if (s > 64) s = 64;
  return s < 1 ? 1 : static_cast<int>(s);
}

constexpr int DIS_TAPS = 75, C2D_TAPS = 49;

int dis_wgrad_slices(int b, int t, int h_o, int w_o, int cout, int cin) {
  return wgrad_slices(static_cast<long long>(b) * t * h_o * w_o, cout, DIS_TAPS * cin);
}

long long dis_wgrad_work_elems(int b, int t, int h_o, int w_o, int cout, int cin) {
  const long long s = dis_wgrad_slices(b, t, h_o, w_o, cout, cin);
  return s * (static_cast<long long>(cout) * DIS_TAPS * cin + cout);
}

long long conv2d_wgrad_work_elems(int n, int h, int w, int cin, int cout) {
  const long long s = wgrad_slices(static_cast<long long>(n) * h * w, cout, C2D_TAPS * cin);
  return s * (static_cast<long long>(cout) * C2D_TAPS * cin + cout);
}

// The GEMM over `slices` K ranges, the bias partials and the ordered reduction (3 or 2 launches).
template <int KT, int KS, int S>
static int run_wgrad(const float* dy, const void* x_hi, const void* x_lo, float* dw, float* db, float* work, int b, int t,
                     int h_in, int w_in, int x_pitch, int x_lead, int cin, int h_o, int w_o, int cout, int pad, int slices,
                     bool bias_rows, cudaStream_t stream) {
  using namespace wgrad;
  constexpr int TAPS = KT * KS * KS;
  static DeviceOnce configured;
  if (const int e = configure_once(configured, SMEM, wgrad_mma_kernel<KT, KS, S>)) return e;
  const long long n_w = static_cast<long long>(cout) * TAPS * cin;
  float* wsb = work + slices * n_w;
  const long long pixels = static_cast<long long>(b) * t * h_o * w_o;
  const dim3 grid((TAPS * cin + NT - 1) / NT, (cout + MT - 1) / MT, slices);
  wgrad_mma_kernel<KT, KS, S><<<grid, THREADS, SMEM, stream>>>(dy, static_cast<const __nv_bfloat16*>(x_hi),
                                                               static_cast<const __nv_bfloat16*>(x_lo), work, b, t, h_in, w_in,
                                                               x_pitch, x_lead, cin, h_o, w_o, cout, pad, slices);
  count_launch();
  if (db) {
    if (bias_rows && cout <= 128)
      bias_partial_rows_kernel<<<slices, 256, 0, stream>>>(dy, wsb, pixels, cout, slices);
    else
      bias_partial_kernel<<<slices, 128, 0, stream>>>(dy, wsb, pixels, cout, slices);
    count_launch();
  }
  reduce_kernel<TAPS><<<static_cast<unsigned>((n_w + 255) / 256), 256, 0, stream>>>(work, wsb, dw, db, cout, cin, slices);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_dis_wgrad(const float* dy, const void* x_hi, const void* x_lo, float* dw, float* db, float* work, int b, int t,
                     int h_in, int w_in, int cin, int h_o, int w_o, int cout, int pad, cudaStream_t stream) {
  return run_wgrad<3, 5, 2>(dy, x_hi, x_lo, dw, db, work, b, t, h_in, w_in, w_in, 0, cin, h_o, w_o, cout, pad,
                            dis_wgrad_slices(b, t, h_o, w_o, cout, cin), false, stream);
}

int launch_conv2d_wgrad(const float* dy, const void* x_hi, const void* x_lo, int x_lead, float* dw, float* db, float* work,
                        int n, int h, int w, int cin, int cout, cudaStream_t stream) {
  const int pitch = x_lead ? conv_rows_pitch(w, x_lead, cin) : w;
  const int slices = wgrad_slices(static_cast<long long>(n) * h * w, cout, C2D_TAPS * cin);
  return run_wgrad<1, 7, 1>(dy, x_hi, x_lo, dw, db, work, n, 1, h, w, pitch, x_lead, cin, h, w, cout, 3, slices, true, stream);
}

}  // namespace e2f
