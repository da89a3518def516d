// Fused modulated deformable convolution (DCNv2, 3x3 / s1 / p1 / d1, Cin=256, Cout=128, 16 deform groups)
// — replaces mmcv.ops.modulated_deform_conv2d as called at model/modules/feat_prop.py:55-58, optionally with
// the offset/mask epilogue of feat_prop.py:41-53 (10*tanh + flow.flip(1), sigmoid) folded into the sampler.
//
// GEMM view: out[M=N*H*W, 128] = A[M, K=2304] * Wp[128, K]^T + bias, where the im2col matrix A is never written
// to global memory: 8 producer warps bilinearly sample x (NHWC fp16, one sample point = 16 channels = 32 B per
// corner) and store fp16 rows straight into the 128B-swizzled K-major shared-memory tile that wgmma reads; the
// packed weight streams in by TMA (SWIZZLE_128B).  The same 8 warps are the two consumer warpgroups (64 rows each):
// the wgmma of K block j runs asynchronously while they sample K block j+1; accumulation is fp32 in registers.
//   K order: k = sp*16 + c,  sp = g*9 + tap  (so offset channels of sp are 2*sp, 2*sp+1 and its mask channel sp)
//   one 64-wide K block = 4 consecutive sample points; 36 K blocks; 4-stage mbarrier ring.
// Roofline (SURVEY §8d): 2*128*2304*M FLOP per call (3.82 GFLOP at M=6480) on the tensor pipe; min bytes
// (x + offset + mask + W + out).
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "dcn_math.cuh"
#include "launch.h"

namespace e2f {
namespace dcn {

// the 16 fp16 channels of one (pixel, deform group) are 32 contiguous, 32-byte aligned bytes in both input layouts
__device__ __forceinline__ void ldg256(const uint4* p, uint4& a, uint4& b) {
  a = __ldg(p);
  b = __ldg(p + 1);
}

constexpr int CIN = 256, COUT = 128, DG = 16, CPG = CIN / DG, TAPS = 9;
constexpr int KTOT = CIN * TAPS;             // 2304
constexpr int NSP = DG * TAPS;               // 144 sample points per output pixel
constexpr int BLOCK_M = 128, BLOCK_K = 64;
constexpr int NUM_KB = KTOT / BLOCK_K;       // 36
constexpr int SP_PER_KB = BLOCK_K / CPG;     // 4
constexpr int STAGES = 4;
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int B_BYTES = COUT * BLOCK_K * 2;
constexpr int PRODUCER_WARPS = 8;                       // 256 threads = 128 rows x 2 pairs of sample points
constexpr int TMA_WARP = PRODUCER_WARPS;
constexpr int THREADS = (PRODUCER_WARPS + 1) * 32;
constexpr int SMEM_BYTES = STAGES * (A_BYTES + B_BYTES) + 256 + 1024;  // + barriers + alignment slack


// GROUPED: x is [N][G][H][W][16] (group-major; the two horizontally adjacent bilinear corners of a sample are one
// contiguous 64 B run -> about half the distinct L1 lines per sample of the NHWC layout [N][H][W][256]).
template <bool FUSED, bool GROUPED, typename OutT>
__global__ void __launch_bounds__(THREADS, 1)
dcn_kernel(const __grid_constant__ CUtensorMap tmap_w, const __half* __restrict__ x,
           const float* __restrict__ offset, const float* __restrict__ mask, const float* __restrict__ head,
           const float2* __restrict__ flow1, const float2* __restrict__ flow2, const float* __restrict__ bias,
           OutT* __restrict__ out, int M, int H, int W, float max_res, __nv_bfloat16* __restrict__ out_hi,
           __nv_bfloat16* __restrict__ out_lo) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* full_a = reinterpret_cast<uint64_t*>(smem + STAGES * (A_BYTES + B_BYTES));
  uint64_t* full_b = full_a + STAGES;
  uint64_t* empty = full_b + STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_a[s], PRODUCER_WARPS);
      mbar_init(&full_b[s], 1);
      mbar_init(&empty[s], PRODUCER_WARPS);
    }
    fence_barrier_init();
  }
  if (warp == TMA_WARP && lane == 0) tma_prefetch_desc(&tmap_w);
  __syncthreads();

  // the TMA warp's branch comes first: with the sampler / MMA warps in the `if` branch and the TMA warp in an `else if`,
  // ptxas serializes every wgmma of the kernel (advisory C7518, WG.DP in divergent path)
  if (warp == TMA_WARP) {
    // ------------------------------------------------------------------ B producer: packed weight via TMA
    if (elect_one()) {   // one thread, chosen by elect.sync: ptxas then emits bare UTCHMMA / UTMALDG (no per-instruction ELECT loop)
      for (int j = 0; j < NUM_KB; ++j) {
        const int stage = j % STAGES;
        const uint32_t phase = (j / STAGES) & 1;
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_b[stage], B_BYTES);
        tma_load_2d(smem_u32(sB + stage * B_BYTES), &tmap_w, &full_b[stage], j * BLOCK_K, 0);
      }
    }
  } else {
    // ------------------------------------------------------------------ A producer: sampler + im2col
    const int r = tid >> 1, s0 = 2 * (tid & 1);          // row, first of this thread's two sample points
    const long long m = static_cast<long long>(blockIdx.x) * BLOCK_M + r;
    const bool row_valid = m < M;
    const long long mm = row_valid ? m : 0;
    const int px = static_cast<int>(mm % W);
    const int py = static_cast<int>((mm / W) % H);
    const long long n = mm / (static_cast<long long>(W) * H);
    const __half* xn = x + n * H * W * CIN;
    constexpr int PIX_STRIDE = GROUPED ? CPG : CIN;      // halfs between horizontally adjacent pixels
    const float* off_p = FUSED ? head + mm * (3 * NSP) : offset + mm * (2 * NSP);
    const float* msk_p = FUSED ? head + mm * (3 * NSP) + 2 * NSP : mask + mm * NSP;
    float2 fl1 = make_float2(0.f, 0.f), fl2 = make_float2(0.f, 0.f);
    if (FUSED) {
      fl1 = __ldg(flow1 + mm);
      fl2 = __ldg(flow2 + mm);
    }
    uint32_t row_off[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) row_off[i] = sw128_offset(r, 2 * s0 + i);
    const int wg = warp >> 2, wq = warp & 3;
    // this warpgroup's 64 A rows start 64 * 128 B into the A tile
    const uint64_t d_a0 = gmma_desc_sw128(smem_u32(sA) + wg * 64 * 128, 16, 1024);
    const uint64_t d_b0 = gmma_desc_sw128(smem_u32(sB), 16, 1024);
    float accf[COUT / 2];

    float2 o_next[2];
    float m_next[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      o_next[u] = __ldg(reinterpret_cast<const float2*>(off_p) + s0 + u);
      m_next[u] = __ldg(msk_p + s0 + u);
    }
    for (int j = 0; j < NUM_KB; ++j) {
      const int stage = j % STAGES;
      const uint32_t phase = (j / STAGES) & 1;
      uint4 vv[4];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int sp = j * SP_PER_KB + s0 + u;
        float2 o = o_next[u];
        float mk = m_next[u];
        if (j + 1 < NUM_KB) {
          o_next[u] = __ldg(reinterpret_cast<const float2*>(off_p) + sp + SP_PER_KB);
          m_next[u] = __ldg(msk_p + sp + SP_PER_KB);
        }
        const int g = sp / TAPS, tap = sp - g * TAPS;
        if (FUSED) {
          // offset = max_res * tanh(o) + flow.flip(1): even channel (dy) gets v, odd (dx) gets u (feat_prop.py:41-50)
          const float2 fl = (sp < NSP / 2) ? fl1 : fl2;
          o.x = fmaf(max_res, fast_tanh(o.x), fl.y);
          o.y = fmaf(max_res, fast_tanh(o.y), fl.x);
          mk = fast_sigmoid(mk);
        }
        const int ti = tap / 3, tj = tap - ti * 3;
        const float h_im = static_cast<float>(py - 1 + ti) + o.x;
        const float w_im = static_cast<float>(px - 1 + tj) + o.y;
        const bool inside = row_valid && (h_im > -1.f) && (w_im > -1.f) && (h_im < static_cast<float>(H)) &&
                            (w_im < static_cast<float>(W));
        float acc[16];
  #pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.f;
        if (inside) {
          const float fy = floorf(h_im), fx = floorf(w_im);
          const float ly = h_im - fy, lx = w_im - fx;
          const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
          const __half* xg = GROUPED ? xn + static_cast<long long>(g) * H * W * CPG : xn + g * CPG;
          uint4 lo[4], hi[4];
          float wgt[4];
  #pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int dy = k >> 1, dx = k & 1;
            const int yy = y0 + dy, xx = x0 + dx;
            const bool in = (yy >= 0) && (yy < H) && (xx >= 0) && (xx < W);
            wgt[k] = in ? (dy ? ly : 1.f - ly) * (dx ? lx : 1.f - lx) * mk : 0.f;
            const int po = min(max(yy, 0), H - 1) * W + min(max(xx, 0), W - 1);
            const uint4* p = reinterpret_cast<const uint4*>(xg + static_cast<long long>(po) * PIX_STRIDE);
            ldg256(p, lo[k], hi[k]);
          }
  #pragma unroll
          for (int k = 0; k < 4; ++k) {
            const __half2* pl = reinterpret_cast<const __half2*>(&lo[k]);
            const __half2* ph = reinterpret_cast<const __half2*>(&hi[k]);
  #pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 a = __half22float2(pl[i]);
              const float2 b = __half22float2(ph[i]);
              acc[2 * i] = fmaf(wgt[k], a.x, acc[2 * i]);
              acc[2 * i + 1] = fmaf(wgt[k], a.y, acc[2 * i + 1]);
              acc[8 + 2 * i] = fmaf(wgt[k], b.x, acc[8 + 2 * i]);
              acc[8 + 2 * i + 1] = fmaf(wgt[k], b.y, acc[8 + 2 * i + 1]);
            }
          }
        }
        uint4& v0 = vv[2 * u];
        uint4& v1 = vv[2 * u + 1];
        v0.x = pack_half2(acc[0], acc[1]);   v0.y = pack_half2(acc[2], acc[3]);
        v0.z = pack_half2(acc[4], acc[5]);   v0.w = pack_half2(acc[6], acc[7]);
        v1.x = pack_half2(acc[8], acc[9]);   v1.y = pack_half2(acc[10], acc[11]);
        v1.z = pack_half2(acc[12], acc[13]); v1.w = pack_half2(acc[14], acc[15]);

      }

      mbar_wait(&empty[stage], phase ^ 1);
      uint8_t* a_tile = sA + stage * A_BYTES;
#pragma unroll
      for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(a_tile + row_off[i]) = vv[i];
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&full_a[stage]);

      // K block j on the tensor pipe (asynchronous: it runs while block j+1 is sampled); block j-1 is then complete
      mbar_wait(&full_a[stage], phase);
      mbar_wait(&full_b[stage], phase);
      const uint64_t da = d_a0 + ((stage * A_BYTES) >> 4), db = d_b0 + ((stage * B_BYTES) >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) wgmma_ss<COUT, true>(accf, da + 2 * k, db + 2 * k, (j | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (j > 0 && lane == 0) mbar_arrive(&empty[(j - 1) % STAGES]);
    }
    wgmma_wait<0>();

    // ------------------------------------------------------------------ epilogue: accumulator fragment -> +bias -> global
    // rows r0 and r0 + 8 of the tile, column pairs 8c + 2(lane % 4)
    const long long r0 = static_cast<long long>(blockIdx.x) * BLOCK_M + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
    for (int c = 0; c < COUT / 8; ++c) {
      const int col = 8 * c + 2 * (lane & 3);
      const float b0 = bias ? __ldg(bias + col) : 0.f, b1 = bias ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long om = r0 + 8 * h;
        if (om >= M) continue;
        const float f0 = accf[4 * c + 2 * h] + b0, f1 = accf[4 * c + 2 * h + 1] + b1;
        if constexpr (sizeof(OutT) == 4) {
          *reinterpret_cast<float2*>(out + om * COUT + col) = make_float2(f0, f1);
          if (out_hi) {
            // bf16 (hi, lo) split of the same values: the operand pair of the backbone conv that consumes the aligned
            // features (feat_prop.py:131-136), so no standalone split pass runs between the DCN and that conv
            const __nv_bfloat162 hb = __floats2bfloat162_rn(f0, f1);
            const float2 hf = __bfloat1622float2(hb);
            const __nv_bfloat162 lb = __floats2bfloat162_rn(f0 - hf.x, f1 - hf.y);
            *reinterpret_cast<__nv_bfloat162*>(out_hi + om * COUT + col) = hb;
            *reinterpret_cast<__nv_bfloat162*>(out_lo + om * COUT + col) = lb;
          }
        } else {
          *reinterpret_cast<uint32_t*>(out + om * COUT + col) = pack_half2(f0, f1);
        }
      }
    }
  }
}

__global__ void pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ wp, int cout, int cin, int dg) {
  const int cpg = cin / dg;
  const long long total = static_cast<long long>(cout) * cin * 9;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int k = static_cast<int>(idx % (cin * 9));
  const int o = static_cast<int>(idx / (cin * 9));
  const int sp = k / cpg, c = k - sp * cpg;
  const int g = sp / 9, tap = sp - g * 9;
  wp[idx] = __float2half_rn(w[(static_cast<long long>(o) * cin + g * cpg + c) * 9 + tap]);
}

// fp32 NHWC sources a [N][H][W][Ca], b [N][H][W][Cb] -> fp16 group-major [N][(Ca+Cb)/16][H][W][16]
// (== torch.cat([a, b], 1).half() of feat_prop.py:126 in the layout the sampler wants); one thread per (group, pixel)
__global__ void __launch_bounds__(256) pack_input_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                         __half* __restrict__ xg, int N, int HW, int Ca, int Cb) {
  const int G = (Ca + Cb) / CPG;
  const long long total = static_cast<long long>(N) * G * HW;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int pix = static_cast<int>(i % HW);
  const int g = static_cast<int>((i / HW) % G);
  const long long n = i / (static_cast<long long>(HW) * G);
  const int c0 = g * CPG;
  const float* src = (c0 < Ca) ? a + (n * HW + pix) * Ca + c0 : b + (n * HW + pix) * Cb + (c0 - Ca);
  uint32_t o[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(src) + j);
    o[2 * j] = pack_half2(v.x, v.y);
    o[2 * j + 1] = pack_half2(v.z, v.w);
  }
  uint4* dst = reinterpret_cast<uint4*>(xg + i * CPG);
  dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
  dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

template <bool FUSED, bool GROUPED, typename OutT>
static int launch_variant(const CUtensorMap& tmap, const void* x, const float* offset, const float* mask,
                          const float* head, const float* flow1, const float* flow2, const float* bias, void* out,
                          int M, int h, int w, float max_res, void* out_hi, void* out_lo, cudaStream_t stream) {
  auto kern = dcn_kernel<FUSED, GROUPED, OutT>;
  static DeviceOnce configured;                    // one per template instantiation, one bit per device
  if (const int e = configure_once(configured, SMEM_BYTES, kern)) return e;
  const unsigned blocks = static_cast<unsigned>((M + BLOCK_M - 1) / BLOCK_M);
  kern<<<blocks, THREADS, SMEM_BYTES, stream>>>(tmap, static_cast<const __half*>(x), offset, mask, head,
                                                reinterpret_cast<const float2*>(flow1),
                                                reinterpret_cast<const float2*>(flow2), bias,
                                                static_cast<OutT*>(out), M, h, w, max_res,
                                                static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo));
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace dcn

int launch_dcn_pack_weight(const float* w, void* w_packed, int cout, int cin, int dg, cudaStream_t stream) {
  const long long total = static_cast<long long>(cout) * cin * 9;
  const int threads = 256;
  dcn::pack_weight_kernel<<<static_cast<unsigned>((total + threads - 1) / threads), threads, 0, stream>>>(
      w, static_cast<__half*>(w_packed), cout, cin, dg);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_dcn(const void* x, const float* offset, const float* mask, const float* head, const float* flow1,
               const float* flow2, const void* w_packed, const float* bias, void* out, int n, int h, int w, int cin,
               int cout, int dg, float max_residue, int out_dtype, int x_grouped, cudaStream_t stream, void* out_hi,
               void* out_lo) {
  using namespace dcn;
  if ((out_hi || out_lo) && (out_dtype != 0 || !out_hi || !out_lo)) {
    set_error("deformable conv: the bf16 split output goes with the fp32 output and needs both halves");
    return -1;
  }
  if (cin != CIN || cout != COUT || dg != DG) {
    set_error("deformable conv is specialised for Cin=256, Cout=128, deform_groups=16 (got %d, %d, %d)", cin, cout,
              dg);
    return -2;
  }
  const long long M = static_cast<long long>(n) * h * w;
  if (M <= 0) return 0;
  if (M > 0x7FFFFFFFLL) {
    set_error("N*H*W too large");
    return -2;
  }
  CUtensorMap tmap;
  const cuuint64_t dims[2] = {KTOT, COUT};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(KTOT) * 2};
  const cuuint32_t box[2] = {BLOCK_K, COUT};
  const cuuint32_t estr[2] = {1, 1};
  if (const int e = encode_tmap(&tmap, w_packed, 2, dims, strides, box, estr, "deformable conv weight",
                                CU_TENSOR_MAP_DATA_TYPE_FLOAT16))
    return e;
  const int Mi = static_cast<int>(M);
#define E2F_DCN_LAUNCH(F, G, T) launch_variant<F, G, T>(tmap, x, offset, mask, head, flow1, flow2, bias, out, Mi, h, w, max_residue, out_hi, out_lo, stream)
  if (head) {
    if (x_grouped) return out_dtype == 1 ? E2F_DCN_LAUNCH(true, true, __half) : E2F_DCN_LAUNCH(true, true, float);
    return out_dtype == 1 ? E2F_DCN_LAUNCH(true, false, __half) : E2F_DCN_LAUNCH(true, false, float);
  }
  if (x_grouped) return out_dtype == 1 ? E2F_DCN_LAUNCH(false, true, __half) : E2F_DCN_LAUNCH(false, true, float);
  return out_dtype == 1 ? E2F_DCN_LAUNCH(false, false, __half) : E2F_DCN_LAUNCH(false, false, float);
#undef E2F_DCN_LAUNCH
}

int launch_dcn_pack_input(const float* a, const float* b, void* xg, int n, int h, int w, int ca, int cb,
                          cudaStream_t stream) {
  const long long total = static_cast<long long>(n) * ((ca + cb) / dcn::CPG) * h * w;
  if (total == 0) return 0;
  const int threads = 256;
  dcn::pack_input_kernel<<<static_cast<unsigned>((total + threads - 1) / threads), threads, 0, stream>>>(
      a, b, static_cast<__half*>(xg), n, h * w, ca, cb);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
