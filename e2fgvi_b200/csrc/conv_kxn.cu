// "kx-in-N" convolution for the layers with FEW OUTPUT CHANNELS: SPyNet's 64 -> 32 and 32 -> 16 7x7 convs
// (model/modules/flow_comp.py:181-215) and the decoder's 64 -> 3 output conv (model/e2fgvi.py:149-150, + tanh :262).
//
// Why: with pixels as the M dimension of the implicit GEMM, every MMA re-reads its A tile from shared memory whatever N
// is, so a conv with Cout = 32 or Cout = 3 leaves the tensor pipe mostly idle.  Here the kernel COLUMN taps go into N
// instead of K:
//     D[(y, xin), (kx, co)] = sum_{ky, c} X[y + ky - pad, xin, c] * W[co, c, ky, kx]          (K = ks * C, N = ks * Cout)
//     out[y, x, co]         = sum_{kx}    D[(y, x + kx - pad), (kx, co)]
// One A tile read now feeds ks times more output columns (N = 224 for 7 x 32: the MMA is math-bound again), the K loop is
// ks times shorter, and the horizontal shift-and-add of the second line is done by the epilogue: a tile is 4 rows x 32
// columns of D; the accumulator columns of one kx at a time are staged in shared memory and every thread adds
// `D[.., x + kx - pad]` of its output pixel.  Cost: the 2 * pad border columns of every 32-column tile are recomputed by
// its neighbour (26 / 32 useful for 7x7, 30 / 32 for 3x3).
// fp32-level accuracy as everywhere: bf16 (hi, lo) operand pairs, D += Ah.Wh + Ah.Wl + Al.Wh, fp32 accumulation.
// Pipeline = conv.cu: persistent CTAs, TMA warp + two consumer warpgroups (64 accumulator rows each, in registers).
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace kxn {

constexpr int BM = 128, BK = 64, TW = 32, TH = 4;
constexpr int A_TILE = BM * BK * 2;
constexpr int CONSUMER_WARPS = 8;                     // two warpgroups x 64 accumulator rows
constexpr int THREADS = (CONSUMER_WARPS + 1) * 32;    // + the TMA warp
// one kx slice of the accumulator, [128 rows][co_pad + 4] fp32 (the +4 keeps row-parallel 16-byte reads conflict-free)
constexpr int KSTAGE_BYTES = 128 * (32 + 4) * 4;
constexpr int EPI_TANH = 1, EPI_NCHW = 2;

constexpr int MAX_SRC = 2;
struct Maps {
  CUtensorMap a_hi[MAX_SRC], a_lo[MAX_SRC], w_hi, w_lo;
};

struct Params {
  int N, H, W, Cout, co_pad, ks, pad, chunks, NB;   // Cout: output channels PER GROUP; NB = ks * co_pad accumulator
                                                    // columns (multiple of 16, <= 256); chunks = K chunks per ky (all sources)
  int groups, cout_total;                           // grouped conv (encoder conv 7, e2fgvi.py:97): tile = (pixels, group)
  int nsrc, cig[MAX_SRC], src_chunks[MAX_SRC];      // channels per group and 64-wide K chunks of each source
  int stage_bytes, stages;     // plain variant: ring of [Ah | Al | Wh | Wl] stages, one per (ky, chunk)
  int a_slot_bytes, a_slots;   // HALO variant: ring of [Ah halo | Al halo] slots, one per chunk: (TH + ks - 1) x 32 pixel rows
  int w_slot_bytes, w_slots;   //               ring of [Wh | Wl] slots, one per (chunk, ky)
  float slope;
  int flags;
  const float* bias;
  const float* residual;          // NHWC fp32 [N][H][W][Cout] or null
  float* out;                     // NHWC fp32 (NCHW with EPI_NCHW) or null
  __nv_bfloat16* out_hi;          // NHWC bf16 split [N][H][W][Cout] or null
  __nv_bfloat16* out_lo;
};

// HALO = true (N <= 112 columns: the A operand dominates the L2 -> SM traffic): instead of one 4-row A box per (ky, chunk),
// ONE box of TH + ks - 1 rows per chunk brings the tile's whole vertical halo; the A tile of tap row ky is rows
// [32*ky, 32*ky + 128) of it — a descriptor start shifted by ky * 4096 B, a multiple of the 1024-byte swizzle atom — and only
// the weights stream per ky through their own ring.  A bytes per tile drop 2x (3x3) to 2.8x (7x7).
template <bool HALO, int KS, int CO_PAD>
__global__ void __launch_bounds__(THREADS, 1) conv_kxn_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p) {
  constexpr int NB = KS * CO_PAD;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int ring_bytes = HALO ? p.a_slots * p.a_slot_bytes + p.w_slots * p.w_slot_bytes : p.stages * p.stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + ring_bytes);      // plain: stage full / HALO: A slot full
  uint64_t* empty = full + 4;
  uint64_t* w_full = empty + 4;                                          // HALO: weight ring
  uint64_t* w_empty = w_full + 4;
  float* bias_s = reinterpret_cast<float*>(smem + ring_bytes + 256);     // [512]
  float* kstage = bias_s + 512;                                          // [128][CO_PAD + 4]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int W_TILE = NB * BK * 2;
  const int step_x = TW - 2 * p.pad;                                   // output columns a tile produces
  const int tiles_x = (p.W + step_x - 1) / step_x, tiles_y = (p.H + TH - 1) / TH;
  const int num_tiles = p.N * tiles_y * tiles_x * p.groups;
  for (int i = tid; i < 512; i += THREADS) bias_s[i] = (p.bias && i < p.cout_total) ? __ldg(p.bias + i) : 0.f;

  if (tid == 0) {
    for (int s = 0; s < 4; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMER_WARPS);
      mbar_init(&w_full[s], 1);
      mbar_init(&w_empty[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
    for (int i = 0; i < p.nsrc; ++i) {
      tma_prefetch_desc(&maps.a_hi[i]);
      tma_prefetch_desc(&maps.a_lo[i]);
    }
    tma_prefetch_desc(&maps.w_hi);
    tma_prefetch_desc(&maps.w_lo);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      if (HALO) {
        const int HR = TH + p.ks - 1;
        const uint32_t a_tx = 2u * static_cast<uint32_t>(HR) * TW * 128u, w_tx = 2u * static_cast<uint32_t>(W_TILE);
        uint8_t* wring = smem + p.a_slots * p.a_slot_bytes;
        uint32_t ia = 0, iw = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          const int g = tile % p.groups, tp = tile / p.groups;
          const int tx = tp % tiles_x, ty = (tp / tiles_x) % tiles_y, n = tp / (tiles_x * tiles_y);
          const int xs = tx * step_x - p.pad, ys = ty * TH - p.pad;     // first D-grid column / first halo row
          int chunk = 0;
          for (int s = 0; s < p.nsrc; ++s)
            for (int j = 0; j < p.src_chunks[s]; ++j, ++chunk, ++ia) {
              const int aslot = ia % p.a_slots;
              mbar_wait(&empty[aslot], ((ia / p.a_slots) & 1) ^ 1);
              mbar_arrive_expect_tx(&full[aslot], a_tx);
              const uint32_t a0 = smem_u32(smem + aslot * p.a_slot_bytes);
              const int c0 = g * p.cig[s] + j * BK;
              tma_load_4d(a0, &maps.a_hi[s], &full[aslot], c0, xs, ys, n);
              tma_load_4d(a0 + HR * TW * 128, &maps.a_lo[s], &full[aslot], c0, xs, ys, n);
              for (int ky = 0; ky < p.ks; ++ky, ++iw) {
                const int wslot = iw % p.w_slots;
                mbar_wait(&w_empty[wslot], ((iw / p.w_slots) & 1) ^ 1);
                mbar_arrive_expect_tx(&w_full[wslot], w_tx);
                const uint32_t w0 = smem_u32(wring + wslot * p.w_slot_bytes);
                const int kb = ky * p.chunks + chunk;
                tma_load_2d(w0, &maps.w_hi, &w_full[wslot], kb * BK, g * p.NB);
                tma_load_2d(w0 + W_TILE, &maps.w_lo, &w_full[wslot], kb * BK, g * p.NB);
              }
            }
        }
      } else {
      const uint32_t stage_tx = 2u * A_TILE + 2u * static_cast<uint32_t>(W_TILE);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int g = tile % p.groups, tp = tile / p.groups;
        const int tx = tp % tiles_x, ty = (tp / tiles_x) % tiles_y, n = tp / (tiles_x * tiles_y);
        const int xs = tx * step_x - p.pad, y0 = ty * TH;              // first D-grid column / row of the tile
        int kb = 0;
        for (int ky = 0; ky < p.ks; ++ky)
          for (int s = 0; s < p.nsrc; ++s)
            for (int j = 0; j < p.src_chunks[s]; ++j, ++kb, ++it) {
              const int stage = it % p.stages;
              mbar_wait(&empty[stage], ((it / p.stages) & 1) ^ 1);
              mbar_arrive_expect_tx(&full[stage], stage_tx);
              const uint32_t s0 = smem_u32(smem + stage * p.stage_bytes);
              // channels past the group's slice (the next group's, or out of bounds = zero) meet zero weights
              const int c0 = g * p.cig[s] + j * BK;
              tma_load_4d(s0, &maps.a_hi[s], &full[stage], c0, xs, y0 + ky - p.pad, n);
              tma_load_4d(s0 + A_TILE, &maps.a_lo[s], &full[stage], c0, xs, y0 + ky - p.pad, n);
              tma_load_2d(s0 + 2 * A_TILE, &maps.w_hi, &full[stage], kb * BK, g * p.NB);
              tma_load_2d(s0 + 2 * A_TILE + W_TILE, &maps.w_lo, &full[stage], kb * BK, g * p.NB);
            }
      }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: wgmma main loop
    // warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) = tile rows 2 wg, 2 wg + 1
    const int wg = warp >> 2, wq = warp & 3;
    float d[NB / 2];
    uint32_t it = 0, ia = 0, iw = 0;
    const uint64_t d_w0 = gmma_desc_sw128(smem_u32(smem + (HALO ? p.a_slots * p.a_slot_bytes : 2 * A_TILE)), 16, 1024);
    const uint64_t d_a0 = gmma_desc_sw128(smem_u32(smem) + wg * 64 * 128, 16, 1024);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      if (HALO) {
        const int HR = TH + p.ks - 1;
        const uint32_t lo_off = static_cast<uint32_t>(HR * TW * 128) >> 4;
        for (int chunk = 0; chunk < p.chunks; ++chunk, ++ia) {
          const int aslot = ia % p.a_slots;
          mbar_wait(&full[aslot], (ia / p.a_slots) & 1);
          const uint64_t d_ah = d_a0 + (static_cast<uint32_t>(aslot * p.a_slot_bytes) >> 4);
          for (int ky = 0; ky < KS; ++ky, ++iw) {
            const int wslot = iw % p.w_slots;
            mbar_wait(&w_full[wslot], (iw / p.w_slots) & 1);
            const uint64_t dah0 = d_ah + ((static_cast<uint32_t>(ky) * TW * 128) >> 4);   // rows [32 ky, 32 ky + 128) of the halo
            const uint64_t dwh0 = d_w0 + (static_cast<uint32_t>(wslot * p.w_slot_bytes) >> 4);
            const uint64_t dwl0 = dwh0 + (static_cast<uint32_t>(W_TILE) >> 4);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
              const uint64_t dah = dah0 + 2 * k, dal = dah0 + lo_off + 2 * k;
              wgmma_ss<NB, false>(d, dal, dwh0 + 2 * k, (chunk | ky | k) != 0);   // small terms first
              wgmma_ss<NB, false>(d, dah, dwl0 + 2 * k, 1);
              wgmma_ss<NB, false>(d, dah, dwh0 + 2 * k, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&w_empty[wslot]);
          }
          if (lane == 0) mbar_arrive(&empty[aslot]);
        }
      } else {
        const int num_kb = KS * p.chunks;
        const uint64_t d_al0 = gmma_desc_adv(d_a0, A_TILE), d_wl0 = gmma_desc_adv(d_w0, W_TILE);
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int stage = it % p.stages;
          mbar_wait(&full[stage], (it / p.stages) & 1);
          const uint32_t soff = static_cast<uint32_t>(stage * p.stage_bytes) >> 4;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            const uint64_t dah = d_a0 + soff + 2 * k, dal = d_al0 + soff + 2 * k;
            const uint64_t dwh = d_w0 + soff + 2 * k, dwl = d_wl0 + soff + 2 * k;
            wgmma_ss<NB, false>(d, dal, dwh, (kb | k) != 0);   // small terms first
            wgmma_ss<NB, false>(d, dah, dwl, 1);
            wgmma_ss<NB, false>(d, dah, dwh, 1);
          }
          wgmma_commit();
          wgmma_wait<1>();                                    // the previous K block's MMAs are done: release its stage
          if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % p.stages]);
        }
        wgmma_wait<0>();
        if (num_kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % p.stages]);
      }

      // ---------------------------------------------------------------- epilogue: warp -> tile row q, lane -> output column
      const int q = warp & 3, half = warp >> 2;               // tile row; first or second half of the 8-channel chunks
      constexpr int CCH = CO_PAD / 16;                        // 8-channel chunks per warp
      const int g = tile % p.groups, tp = tile / p.groups;
      const int tx = tp % tiles_x, ty = (tp / tiles_x) % tiles_y, n = tp / (tiles_x * tiles_y);
      const int cbase = g * p.Cout;                                       // first output channel of the group
      const int CT = p.cout_total;
      const int y = ty * TH + q, x = tx * step_x + lane - p.pad;          // this lane's OUTPUT pixel
      const bool ok = lane >= p.pad && lane < TW - p.pad && y < p.H && x < p.W;
      const size_t pix = (static_cast<size_t>(n) * p.H + y) * p.W + x;
      float accs[CCH][8];
#pragma unroll
      for (int u = 0; u < CCH; ++u)
#pragma unroll
        for (int i = 0; i < 8; ++i) accs[u][i] = 0.f;
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        // stage accumulator columns [kx * CO_PAD, +CO_PAD) of all 128 rows
        const int r = wg * 64 + wq * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
        for (int j = kx * CO_PAD / 8; j < (kx + 1) * CO_PAD / 8; ++j) {
          const int col = 8 * j + c - kx * CO_PAD;
          *reinterpret_cast<float2*>(kstage + r * (CO_PAD + 4) + col) = make_float2(d[4 * j], d[4 * j + 1]);
          *reinterpret_cast<float2*>(kstage + (r + 8) * (CO_PAD + 4) + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int sr = q * 32 + ((lane + kx - p.pad) & 31);       // D column this output needs for tap kx (same tile row)
#pragma unroll
        for (int u = 0; u < CCH; ++u) {
          const float4* s4 = reinterpret_cast<const float4*>(kstage + sr * (CO_PAD + 4) + (half * CCH + u) * 8);
          const float4 a = s4[0], b = s4[1];
          accs[u][0] += a.x; accs[u][1] += a.y; accs[u][2] += a.z; accs[u][3] += a.w;
          accs[u][4] += b.x; accs[u][5] += b.y; accs[u][6] += b.z; accs[u][7] += b.w;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
#pragma unroll
      for (int u = 0; u < CCH; ++u) {
        float* acc = accs[u];
        const int cc = half * CCH + u;
        const int co0 = cc * 8;
        if (ok && co0 < p.Cout) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float a = acc[i] + bias_s[(cbase + co0 + i) & 511];
            a = a > 0.f ? a : a * p.slope;
            if (p.residual && co0 + i < p.Cout) a += __ldg(p.residual + pix * CT + cbase + co0 + i);
            if (p.flags & EPI_TANH) a = tanhf(a);
            acc[i] = a;
          }
          if (p.out) {
            if (p.flags & EPI_NCHW) {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (co0 + i < p.Cout) p.out[((static_cast<size_t>(n) * CT + cbase + co0 + i) * p.H + y) * p.W + x] = acc[i];
            } else if (co0 + 8 <= p.Cout && (CT & 3) == 0 && (cbase & 3) == 0) {
              float4* d4 = reinterpret_cast<float4*>(p.out + pix * CT + cbase + co0);
              d4[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
              d4[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (co0 + i < p.Cout) p.out[pix * CT + cbase + co0 + i] = acc[i];
            }
          }
          if (p.out_hi && co0 + 8 <= p.Cout) {                // split output: Cout % 8 == 0 (checked by the launcher)
            uint32_t hp[4], lp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const __nv_bfloat162 hb = __floats2bfloat162_rn(acc[2 * i], acc[2 * i + 1]);
              const float2 hf = __bfloat1622float2(hb);
              const __nv_bfloat162 lb = __floats2bfloat162_rn(acc[2 * i] - hf.x, acc[2 * i + 1] - hf.y);
              hp[i] = *reinterpret_cast<const uint32_t*>(&hb);
              lp[i] = *reinterpret_cast<const uint32_t*>(&lb);
            }
            *reinterpret_cast<uint4*>(p.out_hi + pix * CT + cbase + co0) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
            *reinterpret_cast<uint4*>(p.out_lo + pix * CT + cbase + co0) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
          }
        }
      }
    }
  }
}

}  // namespace kxn

// sources: nsrc <= 2 NHWC bf16 (hi, lo) tensors with src_c[i] stored channels (multiples of 8; for groups > 1 multiples of
// `groups`); cout = output channels in total (cout / groups <= co_pad per group).  Weights [groups * ks*co_pad rows]
// [ks * chunks * 64] bf16 (hi, lo): row = g*ks*co_pad + kx*co_pad + co, column = (ky*chunks + chunk)*64 + channel with
// the chunks of source 0 first, then source 1 (ops.pack_conv_kxn_weight).
int launch_conv_kxn(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_c, const void* w_hi,
                    const void* w_lo, const float* bias, const float* residual, float* out, void* out_hi, void* out_lo, int n,
                    int h, int w, int cout, int groups, int co_pad, int ks, float slope, int flags, cudaStream_t stream) {
  using namespace kxn;
  const int NB = ks * co_pad, pad = ks / 2;
  if (nsrc < 1 || nsrc > MAX_SRC || groups < 1 || cout % groups || cout > 512) {
    set_error("conv_kxn: nsrc=%d groups=%d cout=%d", nsrc, groups, cout);
    return -2;
  }
  const int cog = cout / groups;
  if ((ks != 3 && ks != 7) || (co_pad != 16 && co_pad != 32) || cog > co_pad) {
    set_error("conv_kxn: unsupported shape (ks=%d cout/groups=%d co_pad=%d): needs ks in {3,7}, co_pad in {16,32}", ks, cog, co_pad);
    return -2;
  }
  if (out_hi && (cog % 8 || cout % 8)) {
    set_error("conv_kxn: split output needs Cout %% 8 == 0 per group");
    return -2;
  }
  Maps maps;
  Params p;
  p.N = n; p.H = h; p.W = w; p.Cout = cog; p.co_pad = co_pad; p.ks = ks; p.pad = pad; p.NB = NB;
  p.groups = groups; p.cout_total = cout; p.nsrc = nsrc;
  p.slope = slope; p.flags = flags; p.bias = bias; p.residual = residual; p.out = out;
  p.out_hi = static_cast<__nv_bfloat16*>(out_hi); p.out_lo = static_cast<__nv_bfloat16*>(out_lo);
  p.chunks = 0;
  for (int i = 0; i < MAX_SRC; ++i) p.cig[i] = p.src_chunks[i] = 0;
  for (int i = 0; i < nsrc; ++i) {
    const int c = src_c[i];
    if (c <= 0 || c % 8 || c % groups) {
      set_error("conv_kxn: source %d has %d channels (needs a multiple of 8 and of groups)", i, c);
      return -2;
    }
    p.cig[i] = c / groups;
    p.src_chunks[i] = (p.cig[i] + BK - 1) / BK;
    p.chunks += p.src_chunks[i];
  }
  const int w_tile = NB * BK * 2;
  p.stage_bytes = 2 * A_TILE + 2 * w_tile;                      // multiple of 1024 (NB % 16 == 0 -> NB*128 % 2048 == 0)
  const int extra = 4096 + KSTAGE_BYTES;                        // barriers, bias, kx staging, alignment
  p.stages = (3 * p.stage_bytes + extra <= 227 * 1024) ? 3 : 2;
  // HALO variant where A dominates the operand traffic and two halo slots + >= 2 weight slots fit
  const int HR = TH + ks - 1;
  p.a_slot_bytes = 2 * HR * TW * 128;
  p.a_slots = 2;
  p.w_slot_bytes = 2 * w_tile;
  p.w_slots = 3;
  // the halo variant pays off for the multi-chunk 3x3 layers; where a tile has ONE chunk no A prefetch across the tile
  // boundary hides behind the 3 or 7 tap rows
  bool halo = NB <= 112 && ks == 3 && p.chunks >= 2;
  if (halo && p.a_slots * p.a_slot_bytes + p.w_slots * p.w_slot_bytes + extra > 227 * 1024) p.w_slots = 2;
  if (halo && p.a_slots * p.a_slot_bytes + p.w_slots * p.w_slot_bytes + extra > 227 * 1024) halo = false;
  if (!halo && p.stages * p.stage_bytes + extra > 227 * 1024) {
    set_error("conv_kxn: stage does not fit in shared memory");
    return -2;
  }
  for (int i = 0; i < nsrc; ++i) {
    const int c = src_c[i];
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(c), static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h), static_cast<cuuint64_t>(n)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(c) * 2, static_cast<cuuint64_t>(w) * c * 2, static_cast<cuuint64_t>(h) * w * c * 2};
    const cuuint32_t box[4] = {BK, TW, static_cast<cuuint32_t>(halo ? HR : TH), 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    for (int part = 0; part < 2; ++part)
      if (const int e = encode_tmap(part ? &maps.a_lo[i] : &maps.a_hi[i], part ? src_lo[i] : src_hi[i], 4, dims, strides, box,
                                    estr, "conv_kxn source"))
        return e;
  }
  {
    const int kcols = ks * p.chunks * BK;
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(kcols), static_cast<cuuint64_t>(groups) * NB};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(kcols) * 2};
    const cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(NB)};
    const cuuint32_t estr[2] = {1, 1};
    for (int part = 0; part < 2; ++part)
      if (const int e = encode_tmap(part ? &maps.w_lo : &maps.w_hi, part ? w_lo : w_hi, 2, dims, strides, box, estr,
                                    "conv_kxn weight"))
        return e;
  }
  static DeviceOnce cfg;
  if (const int e = configure_once(cfg, 227 * 1024, conv_kxn_kernel<false, 3, 16>, conv_kxn_kernel<false, 3, 32>,
                                   conv_kxn_kernel<false, 7, 16>, conv_kxn_kernel<false, 7, 32>, conv_kxn_kernel<true, 3, 16>,
                                   conv_kxn_kernel<true, 3, 32>, conv_kxn_kernel<true, 7, 16>, conv_kxn_kernel<true, 7, 32>))
    return e;
  const int step_x = TW - 2 * pad;
  const long long tiles = static_cast<long long>(n) * ((h + TH - 1) / TH) * ((w + step_x - 1) / step_x) * groups;
  if (tiles == 0) return 0;
  if (tiles > 0x7FFFFFFFLL) {
    set_error("conv_kxn: too many tiles");
    return -2;
  }
  const int grid = tiles < num_sms() ? static_cast<int>(tiles) : num_sms();
  const int smem = (halo ? p.a_slots * p.a_slot_bytes + p.w_slots * p.w_slot_bytes : p.stages * p.stage_bytes) + extra;
  auto kern = halo ? (ks == 3 ? (co_pad == 16 ? conv_kxn_kernel<true, 3, 16> : conv_kxn_kernel<true, 3, 32>)
                              : (co_pad == 16 ? conv_kxn_kernel<true, 7, 16> : conv_kxn_kernel<true, 7, 32>))
                   : (ks == 3 ? (co_pad == 16 ? conv_kxn_kernel<false, 3, 16> : conv_kxn_kernel<false, 3, 32>)
                              : (co_pad == 16 ? conv_kxn_kernel<false, 7, 16> : conv_kxn_kernel<false, 7, 32>));
  kern<<<grid, THREADS, smem, stream>>>(maps, p);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
