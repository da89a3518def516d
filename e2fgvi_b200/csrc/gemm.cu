// Linear layers of the transformer path (nn.Linear at tfocal_transformer.py:44 ss.embedding, :68 sc.embedding,
// :221 attn.qkv, :398 attn.proj, :89/:97 mlp.conv1/conv2) as ONE persistent wgmma GEMM with fp32-level accuracy:
//     out[M,N] = A[M,K] . W[N,K]^T + bias[N] (+ residual[M,N])
// fp32 operands are split into two bf16 terms (x = hi + lo, |lo| <= 2^-9 |x|) and the product is evaluated as
//     Ah.Wh + Ah.Wl + Al.Wh      (the dropped Al.Wl term is ~2^-18 relative)
// on the bf16 tensor pipe with fp32 accumulation — bf16 keeps the full fp32 exponent range, so no scaling is needed.
// Relative error per output ~2^-17, versus 2^-11 for TF32.
//
// Structure (Hopper warp-specialised GEMM): persistent CTAs over a static tile schedule (n fastest, so concurrently
// running CTAs share A row-panels in L2); warp 8 = TMA producer (4 tensor maps: Ah, Al, Wh, Wl, SWIZZLE_128B, K tail /
// row tails zero-filled by TMA); warps 0-7 = two consumer warpgroups, each owning 64 rows of the 128-row tile: 12
// wgmma per 64-wide K block with the accumulator in registers, one K block in flight while the previous stage is
// released, then +bias (+residual) -> fp32/fp16 global store straight from the accumulator fragment.
// Roofline: tensor-bound, 3 x 2*M*N*K bf16 FLOP of tensor work per 2*M*N*K algorithmic fp32 FLOP.
#include <cuda.h>
#include <cstdlib>
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace gemm {

constexpr int BM = 128, BK = 64;
constexpr int A_TILE = BM * BK * 2;                // 16 KB (one bf16 term)
constexpr int CONSUMER_WARPS = 8;                  // two warpgroups x 64 accumulator rows
constexpr int THREADS = (CONSUMER_WARPS + 1) * 32; // + the TMA warp

template <int BN>
struct Cfg {
  static constexpr int W_TILE = BN * BK * 2;
  static constexpr int STAGE = 2 * A_TILE + 2 * W_TILE;
  static constexpr int STAGES = (BN == 128) ? 3 : 2;
  static constexpr int SMEM = STAGES * STAGE + 256 + 1024;
};

template <int BN, typename OutT>
__global__ void __launch_bounds__(THREADS, 1)
linear_kernel(const __grid_constant__ CUtensorMap tm_ah, const __grid_constant__ CUtensorMap tm_al,
              const __grid_constant__ CUtensorMap tm_wh, const __grid_constant__ CUtensorMap tm_wl,
              const float* __restrict__ bias, const float* __restrict__ residual, OutT* __restrict__ out, int M,
              int N, int K) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE);
  uint64_t* empty = full + C::STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  const int num_kb = (K + BK - 1) / BK;
  const int num_items = tiles_m * tiles_n;

  if (tid == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tm_ah);
    tma_prefetch_desc(&tm_al);
    tma_prefetch_desc(&tm_wh);
    tma_prefetch_desc(&tm_wl);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      uint32_t it = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int m0 = (item / tiles_n) * BM, n0 = (item % tiles_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int stage = it % C::STAGES;
          mbar_wait(&empty[stage], ((it / C::STAGES) & 1) ^ 1);
          mbar_arrive_expect_tx(&full[stage], C::STAGE);
          const uint32_t s0 = smem_u32(smem + stage * C::STAGE);
          tma_load_2d(s0, &tm_ah, &full[stage], kb * BK, m0);
          tma_load_2d(s0 + A_TILE, &tm_al, &full[stage], kb * BK, m0);
          tma_load_2d(s0 + 2 * A_TILE, &tm_wh, &full[stage], kb * BK, n0);
          tma_load_2d(s0 + 2 * A_TILE + C::W_TILE, &tm_wl, &full[stage], kb * BK, n0);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: wgmma main loop + epilogue
    const int wg = warp >> 2, wq = warp & 3;
    // stage-0 descriptors (this warpgroup's 64 A rows start 64 * 128 B into the A tiles); stage s / K step k are
    // reached with one 64-bit add each
    const uint64_t d_ah0 = gmma_desc_sw128(smem_u32(smem) + wg * 64 * 128, 16, 1024);
    const uint64_t d_al0 = gmma_desc_adv(d_ah0, A_TILE);
    const uint64_t d_wh0 = gmma_desc_sw128(smem_u32(smem) + 2 * A_TILE, 16, 1024);
    const uint64_t d_wl0 = gmma_desc_adv(d_wh0, C::W_TILE);
    const bool vec_ok = (N & 1) == 0;                         // rows start on 8-byte boundaries
    float acc[BN / 2];
    uint32_t it = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const int m0 = (item / tiles_n) * BM, n0 = (item % tiles_n) * BN;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int stage = it % C::STAGES;
        mbar_wait(&full[stage], (it / C::STAGES) & 1);
        const uint32_t soff = (stage * C::STAGE) >> 4;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t dah = d_ah0 + soff + 2 * k, dal = d_al0 + soff + 2 * k;
          const uint64_t dwh = d_wh0 + soff + 2 * k, dwl = d_wl0 + soff + 2 * k;
          wgmma_ss<BN, false>(acc, dal, dwh, (kb | k) != 0);   // small terms first
          wgmma_ss<BN, false>(acc, dah, dwl, 1);
          wgmma_ss<BN, false>(acc, dah, dwh, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();                                      // the previous K block's MMAs are done: release its stage
        if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % C::STAGES]);
      }
      wgmma_wait<0>();
      if (num_kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % C::STAGES]);
      // fragment: rows r0 and r0 + 8, column pairs 8j + 2(lane % 4)
      const int r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
      const int cb = n0 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = cb + 8 * j;
        if (col >= N) continue;
        const bool pair = vec_ok && col + 1 < N;
        const float b0 = bias ? __ldg(bias + col) : 0.f;
        const float b1 = (bias && col + 1 < N) ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int R = r0 + 8 * h;
          if (R >= M) continue;
          const size_t o = static_cast<size_t>(R) * N + col;
          float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
          if (pair) {
            if (residual) {
              const float2 r2 = __ldg(reinterpret_cast<const float2*>(residual + o));
              v0 += r2.x;
              v1 += r2.y;
            }
            if constexpr (sizeof(OutT) == 4) *reinterpret_cast<float2*>(out + o) = make_float2(v0, v1);
            else *reinterpret_cast<uint32_t*>(out + o) = pack_half2(v0, v1);
          } else {
            if (residual) v0 += __ldg(residual + o);
            if constexpr (sizeof(OutT) == 4) out[o] = v0;
            else out[o] = __float2half_rn(v0);
            if (col + 1 < N) {
              if (residual) v1 += __ldg(residual + o + 1);
              if constexpr (sizeof(OutT) == 4) out[o + 1] = v1;
              else out[o + 1] = __float2half_rn(v1);
            }
          }
        }
      }
    }
  }
}

// x = hi + lo with hi = bf16(x), lo = bf16(x - hi); 8 elements per thread
__global__ void __launch_bounds__(256) split_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                                                         __nv_bfloat16* __restrict__ lo, long long n8) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float4 a = __ldg(reinterpret_cast<const float4*>(x) + 2 * i);
  const float4 b = __ldg(reinterpret_cast<const float4*>(x) + 2 * i + 1);
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  __align__(16) __nv_bfloat16 h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    h[e] = __float2bfloat16_rn(v[e]);
    l[e] = __float2bfloat16_rn(v[e] - __bfloat162float(h[e]));
  }
  reinterpret_cast<uint4*>(hi)[i] = *reinterpret_cast<const uint4*>(h);
  reinterpret_cast<uint4*>(lo)[i] = *reinterpret_cast<const uint4*>(l);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

static int make_map(CUtensorMap* tm, const void* base, int rows, int k, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return -4;
  }
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(k) * 2};
  const cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%d k=%d)", static_cast<int>(r), rows, k);
    return -4;
  }
  return 0;
}

template <int BN, typename OutT>
static int launch_variant(const void* ah, const void* al, const void* wh, const void* wl, const float* bias,
                          const float* residual, void* out, int m, int n, int k, cudaStream_t stream) {
  CUtensorMap tah, tal, twh, twl;
  int st;
  if ((st = make_map(&tah, ah, m, k, BM))) return st;
  if ((st = make_map(&tal, al, m, k, BM))) return st;
  if ((st = make_map(&twh, wh, n, k, BN))) return st;
  if ((st = make_map(&twl, wl, n, k, BN))) return st;
  auto kern = linear_kernel<BN, OutT>;
  static DeviceOnce cfg;
  const int dev = current_device();
  if (!device_done(cfg, dev)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM);
    if (e != cudaSuccess) return static_cast<int>(e);
    device_mark(cfg, dev);
  }
  const int items = ((m + BM - 1) / BM) * ((n + BN - 1) / BN);
  const int grid = items < num_sms() ? items : num_sms();     // persistent: one CTA per SM
  kern<<<grid, THREADS, Cfg<BN>::SMEM, stream>>>(tah, tal, twh, twl, bias, residual, static_cast<OutT*>(out), m, n, k);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace gemm

int launch_split_bf16(const float* x, void* hi, void* lo, long long n, cudaStream_t stream) {
  const long long n8 = n / 8;
  if (n8 == 0) return 0;
  const int threads = 256;
  gemm::split_bf16_kernel<<<static_cast<unsigned>((n8 + threads - 1) / threads), threads, 0, stream>>>(
      x, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), n8);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_linear_bf16x3(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                         const float* residual, void* out, int m, int n, int k, int out_dtype, int block_n,
                         cudaStream_t stream) {
  using namespace gemm;
  if (m == 0 || n == 0) return 0;
  if (block_n == 256)
    return out_dtype == 1 ? launch_variant<256, __half>(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, stream)
                          : launch_variant<256, float>(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, stream);
  return out_dtype == 1 ? launch_variant<128, __half>(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, stream)
                        : launch_variant<128, float>(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, stream);
}

}  // namespace e2f
