// Weight and bias gradients of the transformer's Linear layers (ss.embedding, sc.embedding, mlp.conv1.0, mlp.conv2.1):
//     dW[n][k] = sum over tokens m of dY[m][n] * X[m][k]        db[n] = sum over m of dY[m][n]
// Both operands are token-major, so the reduction runs over the outer index of both.  TMA loads 64-token x 64-column
// boxes of each (128-byte swizzle) and wgmma reads them as MN-major operands (its transpose bits set): nothing is staged
// through registers.  bf16 three-term split (dYl.Xh + dYh.Xl + dYh.Xh) with fp32 accumulation, the accuracy class of
// the forward Linear.
//  * Persistent CTAs over items (slice, n tile, k tile) of 128 x 128 dW tiles; warp 4 fills a ring of 3 x 64 KB stages
//    [dYh | dYl | Xh | Xl] by TMA, warps 0-3 (one warpgroup) run the MMAs, 24 m64n128k16 per 64-token block.
//  * Split-K over the tokens: `slices` contiguous token ranges of whole 64-token blocks, a function of the shape alone.
//    Each item writes its partial tile to the fp32 workspace (or straight to dW when there is one slice) and a second
//    kernel adds the slices in slice order: every sum has a fixed order, so results are bit-identical from run to run.
//  * The bias gradient is read from the dY tiles already in shared memory: the items of k tile 0 sum their 128 columns
//    over the block's 64 tokens (thread = column, tokens in order, hi + lo) while the block's MMAs run.
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace lwgrad {

constexpr int TN = 128, TK = 128, KB = 64;     // dW tile (n x k) and tokens per K block
constexpr int BOX = 64 * KB * 2;               // one 64-column x 64-token bf16 TMA box: 8 KB
constexpr int PART = 2 * BOX;                  // one bf16 term of a 128-column operand tile
constexpr int STAGE = 4 * PART;                // 64 KB
constexpr int STAGES = 3;
constexpr int THREADS = 160;                   // warps 0-3: the consumer warpgroup; warp 4: the TMA producer
constexpr int SMEM = STAGES * STAGE + 256 + 1024;

// token range of a slice: whole K blocks
__host__ __device__ inline long long slice_len(long long m, int slices) {
  const long long per = (m + slices - 1) / slices;
  return (per + KB - 1) / KB * KB;
}

__global__ void __launch_bounds__(THREADS, 1)
linear_wgrad_kernel(const __grid_constant__ CUtensorMap tm_dyh, const __grid_constant__ CUtensorMap tm_dyl,
                    const __grid_constant__ CUtensorMap tm_xh, const __grid_constant__ CUtensorMap tm_xl,
                    float* __restrict__ out, float* __restrict__ out_b, int M, int N, int K, int slices) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE);
  uint64_t* empty = full + STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles_k = (K + TK - 1) / TK;
  const int tiles = ((N + TN - 1) / TN) * tiles_k;
  const int items = tiles * slices;
  const long long len = slice_len(M, slices);

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);                         // the 4 consumer warps
    }
    fence_barrier_init();
    tma_prefetch_desc(&tm_dyh);
    tma_prefetch_desc(&tm_dyl);
    tma_prefetch_desc(&tm_xh);
    tma_prefetch_desc(&tm_xl);
  }
  __syncthreads();

  // item -> slice z, tile origin (n0, k0), token range [m0, m0 + nkb * KB)
  auto decode = [&](int item, int& z, int& n0, int& k0, long long& m0, int& nkb) {
    z = item / tiles;
    const int t = item - z * tiles;
    n0 = (t / tiles_k) * TN;
    k0 = (t % tiles_k) * TK;
    m0 = len * z;
    const long long m1 = m0 + len < M ? m0 + len : M;
    nkb = m0 < m1 ? static_cast<int>((m1 - m0 + KB - 1) / KB) : 0;
  };

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      uint32_t it = 0;
      for (int item = blockIdx.x; item < items; item += gridDim.x) {
        int z, n0, k0, nkb;
        long long m0;
        decode(item, z, n0, k0, m0, nkb);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int stage = it % STAGES;
          mbar_wait(&empty[stage], ((it / STAGES) & 1) ^ 1);
          mbar_arrive_expect_tx(&full[stage], STAGE);
          const uint32_t s0 = smem_u32(smem + stage * STAGE);
          const int m = static_cast<int>(m0) + kb * KB;
          for (int h = 0; h < 2; ++h) {
            tma_load_2d(s0 + h * BOX, &tm_dyh, &full[stage], n0 + 64 * h, m);
            tma_load_2d(s0 + PART + h * BOX, &tm_dyl, &full[stage], n0 + 64 * h, m);
            tma_load_2d(s0 + 2 * PART + h * BOX, &tm_xh, &full[stage], k0 + 64 * h, m);
            tma_load_2d(s0 + 3 * PART + h * BOX, &tm_xl, &full[stage], k0 + 64 * h, m);
          }
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumer warpgroup
  // stage-0 descriptors: A = dY columns [64 h, 64 h + 64) (one atom), B = X's 128 columns (two atoms, LBO = BOX);
  // 8-token groups are 1024 B apart, a k16 step is 2048 B
  const uint32_t sbase = smem_u32(smem);
  const uint64_t d_ah0 = gmma_desc_sw128(sbase, BOX, 1024), d_al0 = gmma_desc_adv(d_ah0, PART);
  const uint64_t d_bh0 = gmma_desc_sw128(sbase + 2 * PART, BOX, 1024), d_bl0 = gmma_desc_adv(d_bh0, PART);
  constexpr uint32_t HALF = BOX >> 4, KSTEP = 2048 >> 4;
  // this thread's bias column inside the dY tile: box tid / 64, column c = tid % 64 (16-byte chunk c / 8, swizzled)
  const uint32_t bcol_box = (tid >> 6) * BOX, bchunk = (tid & 63) >> 3, bword = (tid & 7) * 2;
  float acc[2 * 64];
  uint32_t it = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    int z, n0, k0, nkb;
    long long m0;
    decode(item, z, n0, k0, m0, nkb);
    const bool bias = out_b != nullptr && k0 == 0;
    float bsum = 0.f;
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int stage = it % STAGES;
      mbar_wait(&full[stage], (it / STAGES) & 1);
      const uint32_t soff = (stage * STAGE) >> 4;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KB / 16; ++k) {
        const uint64_t dah = d_ah0 + soff + k * KSTEP, dal = d_al0 + soff + k * KSTEP;
        const uint64_t dbh = d_bh0 + soff + k * KSTEP, dbl = d_bl0 + soff + k * KSTEP;
        wgmma_n128_bf16_tt(acc, dal, dbh, (kb | k) != 0);   // small terms first
        wgmma_n128_bf16_tt(acc + 64, dal + HALF, dbh, (kb | k) != 0);
        wgmma_n128_bf16_tt(acc, dah, dbl, 1);
        wgmma_n128_bf16_tt(acc + 64, dah + HALF, dbl, 1);
        wgmma_n128_bf16_tt(acc, dah, dbh, 1);
        wgmma_n128_bf16_tt(acc + 64, dah + HALF, dbh, 1);
      }
      wgmma_commit();
      if (bias) {
        // column sums of the block's dY (zero-filled past M and N), tokens in order; the stage is held until the
        // arrive below
        const uint32_t hb = sbase + stage * STAGE + bcol_box, lb = hb + PART;
#pragma unroll 8
        for (int r = 0; r < KB; ++r) {
          const uint32_t o = r * 128 + ((bchunk ^ (r & 7)) << 4) + bword;
          unsigned short h, l;
          asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(hb + o));
          asm volatile("ld.shared.u16 %0, [%1];" : "=h"(l) : "r"(lb + o));
          bsum += __bfloat162float(__ushort_as_bfloat16(h)) + __bfloat162float(__ushort_as_bfloat16(l));
        }
      }
      wgmma_wait<1>();                                    // the previous K block's MMAs are done: release its stage
      if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    if (nkb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
    float* dst = out + static_cast<size_t>(z) * N * K;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int n = n0 + 64 * h + 16 * warp + (lane >> 2) + ((i >> 1) & 1) * 8;
        const int k = k0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (n < N && k < K) dst[static_cast<size_t>(n) * K + k] = nkb ? acc[64 * h + i] : 0.f;   // nkb 0: empty slice
      }
    }
    if (bias && n0 + tid < N) out_b[static_cast<size_t>(z) * N + n0 + tid] = bsum;
  }
}

// dW = the slices' partial tiles added in slice order; db likewise
__global__ void __launch_bounds__(256) reduce_kernel(const float* __restrict__ ws, const float* __restrict__ wsb,
                                                     float* __restrict__ dw, float* __restrict__ db, long long total, int n,
                                                     int slices) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) {
    float s = 0.f;
    for (int z = 0; z < slices; ++z) s += ws[static_cast<size_t>(z) * total + i];
    dw[i] = s;
  }
  if (db && i < n) {
    float s = 0.f;
    for (int z = 0; z < slices; ++z) s += wsb[static_cast<size_t>(z) * n + i];
    db[i] = s;
  }
}

static int make_map(CUtensorMap* tm, const void* base, int m, int cols, int pitch) {
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(m)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch) * 2};
  const cuuint32_t box[2] = {64, KB};
  const cuuint32_t estr[2] = {1, 1};
  return encode_tmap(tm, base, 2, dims, strides, box, estr, "linear weight-gradient operand");
}

}  // namespace lwgrad

// Split-K slice count: enough items to fill the GPU about twice at the tile count, at least 4 K blocks per slice, at most
// 64 slices.  A function of the shape alone, so results do not depend on the device.
int linear_wgrad_slices(int m, int n, int k) {
  using namespace lwgrad;
  const long long tiles = static_cast<long long>((n + TN - 1) / TN) * ((k + TK - 1) / TK);
  long long s = (264 + tiles - 1) / tiles;
  const long long cap = static_cast<long long>(m) / (4 * KB);
  if (s > cap) s = cap;
  if (s > 64) s = 64;
  return s < 1 ? 1 : static_cast<int>(s);
}

long long linear_wgrad_work_elems(int m, int n, int k) {
  const long long s = linear_wgrad_slices(m, n, k);
  return s > 1 ? s * (static_cast<long long>(n) * k + n) : 0;
}

int launch_linear_wgrad(const void* dy_hi, const void* dy_lo, int ldy, const void* x_hi, const void* x_lo, int ldx, float* dw,
                        float* db, float* work, int m, int n, int k, cudaStream_t stream) {
  using namespace lwgrad;
  if (m == 0) {                                        // an empty sum
    cudaMemsetAsync(dw, 0, static_cast<size_t>(n) * k * sizeof(float), stream);
    if (db) cudaMemsetAsync(db, 0, static_cast<size_t>(n) * sizeof(float), stream);
    return static_cast<int>(cudaGetLastError());
  }
  CUtensorMap tdyh, tdyl, txh, txl;
  int st;
  if ((st = make_map(&tdyh, dy_hi, m, n, ldy))) return st;
  if ((st = make_map(&tdyl, dy_lo, m, n, ldy))) return st;
  if ((st = make_map(&txh, x_hi, m, k, ldx))) return st;
  if ((st = make_map(&txl, x_lo, m, k, ldx))) return st;
  static DeviceOnce cfg;
  if ((st = configure_once(cfg, SMEM, linear_wgrad_kernel))) return st;
  const int slices = linear_wgrad_slices(m, n, k);
  const long long total = static_cast<long long>(n) * k;
  float* out = slices > 1 ? work : dw;
  float* out_b = db ? (slices > 1 ? work + slices * total : db) : nullptr;
  const int items = ((n + TN - 1) / TN) * ((k + TK - 1) / TK) * slices;
  const int grid = items < num_sms() ? items : num_sms();
  linear_wgrad_kernel<<<grid, THREADS, SMEM, stream>>>(tdyh, tdyl, txh, txl, out, out_b, m, n, k, slices);
  count_launch();
  if (slices > 1) {
    reduce_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(work, work + slices * total, dw, db, total,
                                                                                n, slices);
    count_launch();
  }
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
