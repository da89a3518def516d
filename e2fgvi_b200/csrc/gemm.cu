// Linear layers of the transformer path (nn.Linear at tfocal_transformer.py:44 ss.embedding, :68 sc.embedding,
// :221 attn.qkv, :398 attn.proj, :89/:97 mlp.conv1/conv2) as ONE persistent wgmma GEMM with fp32-level accuracy:
//     out[M,N] = A[M,K] . W[N,K]^T + bias[N] (+ residual[M,N])
// fp32 operands are split into two bf16 terms (x = hi + lo, |lo| <= 2^-9 |x|) and the product is evaluated as
//     Ah.Wh + Ah.Wl + Al.Wh      (the dropped Al.Wl term is ~2^-18 relative)
// on the bf16 tensor pipe with fp32 accumulation — bf16 keeps the full fp32 exponent range, so no scaling is needed.
// Relative error per output ~2^-17, versus 2^-11 for TF32.
//
// Structure (Hopper warp-specialised "ping-pong" GEMM): persistent CTAs over a static schedule of 128 x 128 output
// tiles (n fastest, so concurrently running CTAs share A row-panels in L2).  Warps 8-11 = producer warpgroup; one of
// its threads fills ONE ring of 3 x 64 KB stages [Ah | Al | Wh | Wl] by TMA (SWIZZLE_128B, K tail / row tails
// zero-filled by TMA) in tile order.  Warps 0-7 = two consumer warpgroups that take alternate tiles of the CTA's
// schedule; each owns its whole tile, 128 fp32 accumulators per thread (two m64n128 halves), 6 wgmma per k16 step.
// Two named barriers make the warpgroups issue their main loops in turn, so while one runs tile i's MMAs the other
// runs tile i - 1's epilogue and the tensor pipe never waits for stores.  The epilogue adds bias (staged in shared memory) and the residual and writes through a
// per-warp swizzled buffer, 64 contiguous bytes of a row per store.
// Roofline: tensor-bound, 3 x 2*M*N*K bf16 FLOP of tensor work per 2*M*N*K algorithmic fp32 FLOP.
#include <cuda.h>
#include <cstdlib>
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace gemm {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int A_TILE = BM * BK * 2;                // 16 KB (one bf16 term)
constexpr int W_TILE = BN * BK * 2;                // 16 KB
constexpr int STAGE = 2 * A_TILE + 2 * W_TILE;     // 64 KB
constexpr int STAGES = 3;
constexpr int CONSUMER_WARPS = 8;                  // two warpgroups, one 128 x 128 tile each
constexpr int THREADS = (CONSUMER_WARPS + 4) * 32; // + the producer warpgroup (one thread issues the TMA loads)
// register split (setmaxnreg): 128 accumulators + the epilogue do not fit the 168 registers a 384-thread CTA starts
// with, so the producer warpgroup gives its share to the consumers: 128 x 40 + 256 x 232 <= 64 K
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int EPI_STAGE = 2048;                    // per consumer warp: the epilogue's store-transposition buffer
// stages, epilogue buffers, one tile's bias per warpgroup, mbarriers, alignment slack: 210 KB of the 227 KB
constexpr int SMEM = STAGES * STAGE + CONSUMER_WARPS * EPI_STAGE + 2 * BN * 4 + 256 + 1024;
// named barriers (0 is __syncthreads): ORDER_BAR + w = "warpgroup w may issue its next main loop", 256 threads;
// EPI_BAR + w = warpgroup w alone, 128 threads
constexpr int ORDER_BAR = 1, EPI_BAR = 3;

// Epilogue of the calling warp's 16 rows [row0, row0 + 16) x the tile's 128 columns from n0, read from the warp's
// fragments `acc` of one m64n128 accumulator: out = acc + bias (+ residual), fp32 or fp16.  bias_s = the tile's 128
// bias values in shared memory (zeros when the layer has none).  Each 32-column chunk goes through `stage`, 2 KB
// private to the warp, as in conv.cu's epilogue_tile:
//  1. fragments -> [16 rows][32 fp32], 16-byte chunk q of row a at q ^ (a & 7);
//  2. read back row-wise: lane = (row lane % 16, columns 16 (lane / 16) .. + 16 of the chunk), so bias and residual
//     are 16-byte loads;
//  3. the results go to 64-byte buffer rows through a conflict-free XOR swizzle (fp32: buffer row `lane` = its 16
//     values; fp16: buffer row p = the 32 values of row p), and 4 consecutive lanes store one buffer row: 64
//     contiguous bytes of one output row per store.
// A chunk that runs past N takes a direct per-element path.
template <typename OutT>
__device__ __forceinline__ void epilogue_rows(const float* acc, int row0, int n0, int M, int N,
                                              const float* __restrict__ bias_s, const float* __restrict__ residual,
                                              OutT* __restrict__ out, uint8_t* __restrict__ stage) {
  const int lane = threadIdx.x & 31;
  const int hf = lane >> 4;                            // which 16 columns of a 32-column chunk this lane handles
  const int r = row0 + (lane & 15);                    // this lane's row
  const uint32_t sbase = smem_u32(stage);
  const int sub = lane & 3, prow = lane >> 2;
  // logical 16-byte chunk cc of buffer row rr sits at physical chunk cc ^ ((rr >> 1) & 3); on the read side lanes
  // 4k..4k+3 fetch the 4 chunks of buffer row jr*8 + k.  Both sides touch 8 distinct bank groups per quarter-warp.
  auto st_chunk = [&](int rr, int cc, uint32_t a, uint32_t b, uint32_t c2, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + rr * 64 + ((cc ^ ((rr >> 1) & 3)) << 4)),
                 "r"(a), "r"(b), "r"(c2), "r"(d)
                 : "memory");
  };
  auto ld_chunk = [&](int rr) {
    uint4 u;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                 : "r"(sbase + rr * 64 + ((sub ^ ((rr >> 1) & 3)) << 4))
                 : "memory");
    return u;
  };
#pragma unroll                                         // compile-time fragment indices: acc stays in registers
  for (int c = 0; c < BN / 32; ++c) {
    // ---------------------------------------------------------------- 1 + 2: fragments -> row-wise values
    __syncwarp();                                      // the previous chunk's stores have read the buffer
    const int qa = lane >> 2, qc = (lane & 3) >> 1, qo = (lane & 1) * 8;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * c + jj;                        // columns 8j + 2 (lane % 4) + {0, 1} of rows qa, qa + 8
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(sbase + sw128_offset(qa, 2 * jj + qc) + qo),
                   "f"(acc[4 * j]), "f"(acc[4 * j + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(sbase + sw128_offset(qa + 8, 2 * jj + qc) + qo),
                   "f"(acc[4 * j + 2]), "f"(acc[4 * j + 3]) : "memory");
    }
    __syncwarp();
    uint32_t v[16];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(v[4 * q]), "=r"(v[4 * q + 1]), "=r"(v[4 * q + 2]), "=r"(v[4 * q + 3])
                   : "r"(sbase + sw128_offset(lane & 15, 4 * hf + q))
                   : "memory");
    __syncwarp();                                      // every lane has its values before the buffer is reused
    const int cl = c * 32 + 16 * hf;                   // tile-local first column of this lane's 16
    const int co_chunk = n0 + c * 32, co = n0 + cl;
    if (co_chunk + 32 <= N) {
      // ------------------------------------------------------------ 3: staged, coalesced stores (warp-uniform branch)
      float f[16];
#pragma unroll
      for (int g4 = 0; g4 < 4; ++g4) {
        const float4 b = *reinterpret_cast<const float4*>(bias_s + cl + g4 * 4);
        f[g4 * 4] = __uint_as_float(v[g4 * 4]) + b.x;
        f[g4 * 4 + 1] = __uint_as_float(v[g4 * 4 + 1]) + b.y;
        f[g4 * 4 + 2] = __uint_as_float(v[g4 * 4 + 2]) + b.z;
        f[g4 * 4 + 3] = __uint_as_float(v[g4 * 4 + 3]) + b.w;
      }
      if (residual && r < M) {
        const float4* r4 = reinterpret_cast<const float4*>(residual + static_cast<size_t>(r) * N + co);
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          const float4 ra = __ldg(r4 + g4);
          f[g4 * 4] += ra.x; f[g4 * 4 + 1] += ra.y; f[g4 * 4 + 2] += ra.z; f[g4 * 4 + 3] += ra.w;
        }
      }
      if constexpr (sizeof(OutT) == 4) {
        // buffer row rr = row row0 + rr % 16, columns 16 (rr / 16) .. + 16 of the chunk
#pragma unroll
        for (int cc = 0; cc < 4; ++cc)
          st_chunk(lane, cc, __float_as_uint(f[cc * 4]), __float_as_uint(f[cc * 4 + 1]), __float_as_uint(f[cc * 4 + 2]),
                   __float_as_uint(f[cc * 4 + 3]));
        __syncwarp();
#pragma unroll
        for (int jr = 0; jr < 4; ++jr) {
          const int rr = jr * 8 + prow, row = row0 + (rr & 15);
          const uint4 u = ld_chunk(rr);
          if (row < M)
            *reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * N + co_chunk + 16 * (rr >> 4) + sub * 4) = u;
        }
      } else {
        // buffer row p = the 32 fp16 values of row row0 + p; this lane's 16 are its chunks 2 hf, 2 hf + 1
        uint32_t hp[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) hp[i] = pack_half2(f[2 * i], f[2 * i + 1]);
        st_chunk(lane & 15, 2 * hf, hp[0], hp[1], hp[2], hp[3]);
        st_chunk(lane & 15, 2 * hf + 1, hp[4], hp[5], hp[6], hp[7]);
        __syncwarp();
#pragma unroll
        for (int jr = 0; jr < 2; ++jr) {
          const int rr = jr * 8 + prow, row = row0 + rr;
          const uint4 u = ld_chunk(rr);
          if (row < M) *reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * N + co_chunk + sub * 8) = u;
        }
      }
    } else if (r < M) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int col = co + i;
        if (col < N) {
          const size_t o = static_cast<size_t>(r) * N + col;
          float a = __uint_as_float(v[i]) + bias_s[cl + i];
          if (residual) a += __ldg(residual + o);
          if constexpr (sizeof(OutT) == 4) out[o] = a;
          else out[o] = __float2half_rn(a);
        }
      }
    }
  }
}

template <typename OutT>
__global__ void __launch_bounds__(THREADS, 1)
linear_kernel(const __grid_constant__ CUtensorMap tm_ah, const __grid_constant__ CUtensorMap tm_al,
              const __grid_constant__ CUtensorMap tm_wh, const __grid_constant__ CUtensorMap tm_wl,
              const float* __restrict__ bias, const float* __restrict__ residual, OutT* __restrict__ out, int M,
              int N, int K) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* epi_stage = smem + STAGES * STAGE;
  float* bias_s = reinterpret_cast<float*>(epi_stage + CONSUMER_WARPS * EPI_STAGE);   // [warpgroup][BN]
  uint64_t* full = reinterpret_cast<uint64_t*>(bias_s + 2 * BN);
  uint64_t* empty = full + STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  const int num_kb = (K + BK - 1) / BK;
  const int num_items = tiles_m * tiles_n;
  // this CTA's tiles: item blockIdx.x + i * gridDim.x for i < my_items; warpgroup w takes i = w, w + 2, ...
  const int grid = static_cast<int>(gridDim.x);
  const int my_items = (num_items - static_cast<int>(blockIdx.x) + grid - 1) / grid;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);                         // the 4 warps of the warpgroup that consumed the stage
    }
    fence_barrier_init();
    tma_prefetch_desc(&tm_ah);
    tma_prefetch_desc(&tm_al);
    tma_prefetch_desc(&tm_wh);
    tma_prefetch_desc(&tm_wl);
  }
  __syncthreads();

  if (warp >= CONSUMER_WARPS) {
    // ------------------------------------------------------------------ TMA producer: one ring, in tile order
    regs_dec<PRODUCER_REGS>();
    if (warp == CONSUMER_WARPS && elect_one()) {
      uint32_t it = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int m0 = (item / tiles_n) * BM, n0 = (item % tiles_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int stage = it % STAGES;
          mbar_wait(&empty[stage], ((it / STAGES) & 1) ^ 1);
          mbar_arrive_expect_tx(&full[stage], STAGE);
          const uint32_t s0 = smem_u32(smem + stage * STAGE);
          tma_load_2d(s0, &tm_ah, &full[stage], kb * BK, m0);
          tma_load_2d(s0 + A_TILE, &tm_al, &full[stage], kb * BK, m0);
          tma_load_2d(s0 + 2 * A_TILE, &tm_wh, &full[stage], kb * BK, n0);
          tma_load_2d(s0 + 2 * A_TILE + W_TILE, &tm_wl, &full[stage], kb * BK, n0);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: ping-pong main loop + epilogue
    regs_inc<CONSUMER_REGS>();
    const int wg = warp >> 2, wq = warp & 3;
    // stage-0 descriptors; stage s / K step k / the second 64-row half of the A tiles are reached with one 64-bit add
    const uint64_t d_ah0 = gmma_desc_sw128(smem_u32(smem), 16, 1024);
    const uint64_t d_al0 = gmma_desc_adv(d_ah0, A_TILE);
    const uint64_t d_wh0 = gmma_desc_sw128(smem_u32(smem) + 2 * A_TILE, 16, 1024);
    const uint64_t d_wl0 = gmma_desc_adv(d_wh0, W_TILE);
    constexpr uint32_t HALF = (64 * 128) >> 4;
    float* my_bias = bias_s + wg * BN;
    uint8_t* my_stage = epi_stage + warp * EPI_STAGE;
    float acc[2 * 64];                                  // rows [0, 64) of the tile, then rows [64, 128)
    for (int i = wg; i < my_items; i += 2) {
      const int item = static_cast<int>(blockIdx.x) + i * grid;
      const int m0 = (item / tiles_n) * BM, n0 = (item % tiles_n) * BN;
      const int bcol = n0 + (tid & 127);                 // this thread stages the bias of column bcol
      const float bval = (bias && bcol < N) ? __ldg(bias + bcol) : 0.f;
      // wait for the turn: the other warpgroup has issued tile i - 1's main loop.  All 128 threads of this
      // warpgroup reach this barrier only after their previous epilogue, so my_bias may be overwritten after it.
      if (i > 0) named_sync(ORDER_BAR + wg, 256);
      uint32_t it = static_cast<uint32_t>(i) * num_kb;   // ring position of the tile's first K block
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int stage = it % STAGES;
        mbar_wait(&full[stage], (it / STAGES) & 1);
        const uint32_t soff = (stage * STAGE) >> 4;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t dah = d_ah0 + soff + 2 * k, dal = d_al0 + soff + 2 * k;
          const uint64_t dwh = d_wh0 + soff + 2 * k, dwl = d_wl0 + soff + 2 * k;
          wgmma_ss<BN, false>(acc, dal, dwh, (kb | k) != 0);   // small terms first
          wgmma_ss<BN, false>(acc + 64, dal + HALF, dwh, (kb | k) != 0);
          wgmma_ss<BN, false>(acc, dah, dwl, 1);
          wgmma_ss<BN, false>(acc + 64, dah + HALF, dwl, 1);
          wgmma_ss<BN, false>(acc, dah, dwh, 1);
          wgmma_ss<BN, false>(acc + 64, dah + HALF, dwh, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();                                      // the previous K block's MMAs are done: release its stage
        if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
      }
      if (i + 1 < my_items) named_arrive(ORDER_BAR + (wg ^ 1), 256);   // the other warpgroup may issue tile i + 1
      wgmma_wait<0>();
      if (num_kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
      my_bias[tid & 127] = bval;
      named_sync(EPI_BAR + wg, 128);                        // the tile's bias is in shared memory
      epilogue_rows<OutT>(acc, m0 + wq * 16, n0, M, N, my_bias, residual, out, my_stage);
      epilogue_rows<OutT>(acc + 64, m0 + 64 + wq * 16, n0, M, N, my_bias, residual, out, my_stage);
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

static int make_map(CUtensorMap* tm, const void* base, int rows, int k, int box_rows) {
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(k) * 2};
  const cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  return encode_tmap(tm, base, 2, dims, strides, box, estr, "linear operand");
}

template <typename OutT>
static int launch_variant(const void* ah, const void* al, const void* wh, const void* wl, const float* bias,
                          const float* residual, void* out, int m, int n, int k, cudaStream_t stream) {
  CUtensorMap tah, tal, twh, twl;
  int st;
  if ((st = make_map(&tah, ah, m, k, BM))) return st;
  if ((st = make_map(&tal, al, m, k, BM))) return st;
  if ((st = make_map(&twh, wh, n, k, BN))) return st;
  if ((st = make_map(&twl, wl, n, k, BN))) return st;
  auto kern = linear_kernel<OutT>;
  static DeviceOnce cfg;
  if ((st = configure_once(cfg, SMEM, kern))) return st;
  const int items = ((m + BM - 1) / BM) * ((n + BN - 1) / BN);
  const int grid = items < num_sms() ? items : num_sms();     // persistent: one CTA per SM
  kern<<<grid, THREADS, SMEM, stream>>>(tah, tal, twh, twl, bias, residual, static_cast<OutT*>(out), m, n, k);
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
                         const float* residual, void* out, int m, int n, int k, int out_dtype, cudaStream_t stream) {
  using namespace gemm;
  if (m == 0 || n == 0) return 0;
  return out_dtype == 1 ? launch_variant<__half>(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, stream)
                        : launch_variant<float>(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, stream);
}

}  // namespace e2f
