// 3x3 / stride 1 / pad 1 convolutions of the path (encoder e2fgvi.py:75-109, decoder :143-150, offset heads
// feat_prop.py:20-28, backbones :73-77) as an implicit GEMM on wgmma with fp32-level accuracy (bf16 3-term split,
// see gemm.cu):   out[n,y,x,co] = act( sum_{tap,src,c} X_src[n, y+r-1, x+s-1, c] * W[co, tap, src, c] + b[co] ) (+ res)
//
//  * im2col is done by TMA: activations are NHWC bf16 (hi, lo); one 4-D box {64 ch, 16 x, 8 y, 1 n} per (tap, source,
//    64-channel chunk) lands directly as a 128-row K-major SWIZZLE_128B operand tile; negative / overflowing
//    coordinates are zero-filled by the TMA unit == the conv's zero padding.  Nothing is materialised.
//  * multi-source K: the channel concatenations in front of these convs (torch.cat at e2fgvi.py:103-108,
//    feat_prop.py:36,125,131-136) are never built — each concatenated tensor is its own TMA source.
//  * groups (encoder convs with groups 2/4/8): a tile's N range lives inside one group and its K chunks start at the
//    group's channel offset of every source; chunks that spill past a group's slice hit zero weights.
//  * small-channel sources (cin = 4 / 8 / 16 / 32: SPyNet's 7x7 convs, the 3-channel stem): "window-packed" K.  The
//    source is stored row-gapped, [N][H][W + pad][cin] with `pad` zero pixels in front of every row (the gap doubles
//    as the previous row's right padding).  The tensor map's pixel dimension has a stride of ONE pixel (x conv
//    stride) but dimension 0 spans 64 elements = 64/cin consecutive pixels, so every TMA row is the sliding window
//    [x - pad + g*PX, +PX) x cin — a whole slice of the kernel row per 64-wide K chunk instead of one tap padded from
//    cin to 64 channels (7x fewer K chunks for SPyNet's first conv, 12x for the stem).  Weights for taps past the
//    kernel width are zero; what those positions read is finite data of the same buffer.
//  * epilogue: + bias, LeakyReLU(slope), optional residual add, fp32 NHWC store and/or the bf16 (hi, lo) split of
//    the result — dense NHWC or row-gapped for a following window-packed conv (the zero gaps are written here).
// Pipeline ("ping-pong", as gemm.cu): persistent CTAs; a producer warpgroup whose one thread fills the TMA ring in the
// CTA's tile order, and two consumer warpgroups that take alternate tiles, each owning a whole 128 x BN tile (two
// m64nBN halves, fp32 in registers).  Named barriers make them issue their main loops in turn, so one warpgroup's
// epilogue runs while the other's MMAs keep the tensor pipe busy.  Each warp's epilogue reads its own accumulator
// fragments (no CTA-wide staging tile, so the pipeline gets that room).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstring>
#include "common.cuh"
#include "launch.h"

namespace e2f {
namespace conv {

constexpr int BM = 128, BK = 64;
constexpr int TILE_H = 8, TILE_W = 16;                  // 8 x 16 output pixels = 128 GEMM rows
constexpr int A_TILE = BM * BK * 2;
constexpr int EPI_WARPS = 8;                             // two consumer warpgroups; in the epilogue each warp stores 16-row slices
constexpr int MAX_COUT = 512;                            // bias staged in shared memory once per CTA
constexpr int EPI_STAGE = 2048;                          // per epilogue warp: 32 rows x 64 bytes store-transposition buffer
constexpr int THREADS = (EPI_WARPS + 4) * 32;            // + the producer warpgroup (one thread issues the TMA loads)
// register split (setmaxnreg): two m64nBN accumulators (128 fp32 at BN = 128) + the epilogue do not fit the 168
// registers a 384-thread CTA starts with, so the producer warpgroup gives its share to the consumers: 128 x 40 + 256 x
// 232 <= 64 K
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
// named barriers (0 is __syncthreads): ORDER_BAR + w = "warpgroup w may issue its next main loop", 256 threads
constexpr int ORDER_BAR = 1;
constexpr int MAX_SRC = 4;
constexpr int MAX_TAPS = 80;                             // the discriminator's 3x5x5 kernels list 75 taps

// N tile: 128 output channels; 64 / 32 for the layers with <= 64 / <= 32 output channels per group (decoder, encoder
// conv 1, SPyNet, the 3-channel output conv), which would otherwise waste most of every MMA; 96 for the encoder's
// groups-of-96 conv (e2fgvi.py:86: 768 -> 384, groups 4), where a 128-wide tile would compute 25 % padding.
template <int BN>
struct Cfg {
  static constexpr int W_TILE = BN * BK * 2;
  static constexpr int STAGE = 2 * A_TILE + 2 * W_TILE;   // 64 KB (BN=128) / 56 KB (BN=96) / 48 KB (BN=64) / 40 KB (BN=32)
  // as many stages as fit in the 227 KB a CTA may use: 211 / 168 / 211 / 219 KB
  static constexpr int STAGES = (BN >= 96) ? 3 : (BN == 64) ? 4 : 5;
  static constexpr int SMEM = STAGES * STAGE + 256 + MAX_COUT * 4 + EPI_WARPS * EPI_STAGE + 1024;
};

struct Maps {
  CUtensorMap a_hi[MAX_SRC], a_lo[MAX_SRC], w_hi, w_lo;
};

struct Params {
  int N, H, W, Cout, groups;     // H, W: OUTPUT spatial size
  int ks, stride, pad;           // square kernel size (3 or 7), stride (1 or 2), zero padding
  int nsrc;
  int rows_px;             // 0: dense NHWC sources.  > 0: window-packed K, 64 / cin pixels per K chunk (one source)
  int rows_g;              // ... K chunks per kernel row = ceil(ks / rows_px)
  int out_lead, out_pitch; // split output rows: `out_lead` zero pixels, then W pixels; out_pitch = W + out_lead
  int out_tail;            // zero pixels after the last row of the split output (0 when dense)
  int cig[MAX_SRC];        // channels per group of each source
  int chunks[MAX_SRC];     // ceil(cig / 64)
  int chunks_total;        // sum of chunks
  // Tap table ("gather conv"): tap i reads the input at (y*stride + tap_dy[i], x*stride + tap_dx[i]); a plain k x k conv
  // lists its k*k taps with dy = ky - pad, dx = kx - pad.  Taps are grouped into PHASES: phase ph owns taps
  // [ph_tap0[ph], ph_tap0[ph+1]) and writes output pixel (y*ostep + ph_oy[ph], x*ostep + ph_ox[ph]) of an
  // out_H x out_W image — one phase for a conv; nine for the transposed 7x7 / stride-3 conv that SoftComp's
  // Linear + fold is (tfocal_transformer.py:65-72): output pixels with the same (y mod 3, x mod 3) share a tap set.
  int tile_w, tile_h;      // GEMM-grid pixels per tile (tile_w * tile_h <= 128; rows beyond are idle)
  int nphase, ostep, out_H, out_W;
  long long out_nstride;   // pixels between consecutive images of the fp32 output / residual (dense: out_H * out_W)
  long long osp_nstride;   // ... of the split outputs (dense: out_H * out_pitch)
  int8_t tap_dy[MAX_TAPS], tap_dx[MAX_TAPS];
  uint8_t ph_tap0[10], ph_oy[9], ph_ox[9];
  // 3-D convs (the T3 instantiations, NDHWC activations): image index n = b * t_out + t over OUTPUT frames.  Dense
  // sources: tap i also reads frame t + tap_dt[i].  Window-packed source: kt temporal taps, tap k reads frame
  // t * tstride - tpad + k.  Frames outside [0, T) are zero-filled by the TMA unit (the conv's temporal padding).
  int t_out, kt, tstride, tpad;
  int8_t tap_dt[MAX_TAPS];
  int out_cs;              // channels per pixel of the fp32 / split outputs: Cout, or more for a channel slice
  float slope;             // LeakyReLU negative slope (1 = identity)
  int epi_flags;           // EPI_TANH: tanh after the activation; EPI_NCHW: fp32 output stored [N][Cout][out_H][out_W]
  const float* bias;
  const float* bias_map;   // optional fp32 [out_H][out_W][Cout] added per output pixel (folded Linear bias + sc.bias) or null
  const float* residual;   // NHWC fp32 [N][out_H][out_W][Cout] or null
  float* out;              // NHWC fp32 or null
  __nv_bfloat16* out_hi;   // NHWC bf16 split of the result (operand format of the next conv) or null
  __nv_bfloat16* out_lo;
  // T3 and the DACT instantiations only: derivative of the LeakyReLU(dact_slope) that produced `dact` (bf16, the hi part
  // of the saved activation, Cout channels per pixel; pixel (n, y, x) at n * dact_nstride + y * dact_pitch + dact_lead
  // + x: dense or row-gapped).  The result is multiplied by 1 where dact > 0, else by dact_slope (LeakyReLU keeps the
  // sign of its input, so its output decides).  Null: no multiply.  With a residual the epilogue computes
  // (acc + residual) * derivative: the input gradient of a tensor that several convs read (the encoder's x0) adds the
  // other convs' contributions before the derivative of the activation that produced it.
  const __nv_bfloat16* dact;
  float dact_slope;
  int dact_pitch, dact_lead;
  long long dact_nstride;
};

constexpr int EPI_TANH = 1, EPI_NCHW = 2;     // both only on the element-wise store path (Cout % 4 != 0: the 3-channel output conv)

struct TileCoord {
  int n, y0, x0, g, co0;   // co0: first output channel of the tile (global index)
  int ph, oy, ox;          // phase and its output-pixel offset
};

template <int BN>
__device__ __forceinline__ TileCoord decode_tile(int tile, const Params& p, int tiles_y, int tiles_x, int tiles_ng) {
  TileCoord t;
  const int nt = tile % tiles_ng;
  int r = tile / tiles_ng;
  t.g = r % p.groups;
  r /= p.groups;
  t.ph = r % p.nphase;
  r /= p.nphase;
  const int tx = r % tiles_x;
  r /= tiles_x;
  const int ty = r % tiles_y;
  t.n = r / tiles_y;
  t.y0 = ty * p.tile_h;
  t.x0 = tx * p.tile_w;
  t.co0 = t.g * (p.Cout / p.groups) + nt * BN;
  t.oy = p.ph_oy[t.ph];
  t.ox = p.ph_ox[t.ph];
  return t;
}

// Epilogue of the calling warp's 16 accumulator rows [row0, row0 + 16) x all BN channels of one 128-pixel tile, read
// straight from the wgmma fragments `acc`: + bias, LeakyReLU, optional residual, fp32 and/or bf16-split NHWC stores.
// TW = tile width in pixels (row R is pixel (y0 + R / TW, x0 + R % TW)).  bias_s = the layer's bias in SHARED memory
// (zeros when the layer has none): per-channel __ldg's would queue behind the epilogue's own stores.
//
// Everything goes through `stage`, 2 KB of shared memory private to the warp, one 32-channel chunk at a time:
//  1. fragments -> [16 rows][32 fp32], 16-byte chunk q of row a at q ^ (a & 7): each lane quad holds 8 channels of rows a
//     and a + 8, and the 8 rows of one store instruction hit 8 different bank groups;
//  2. read back row-wise: lane = (row lane % 16, channels 16 (lane / 16) .. + 16 of the chunk), the thread = pixel form
//     in which bias, residual and bias map are 16-byte loads;
//  3. coalesced stores: with thread = pixel, a direct 16-byte store per thread hits 32 different 128-byte lines per
//     instruction (pixels are Cout * 2 or 4 bytes apart), ~125 cycles each.  The results instead go to 64-byte buffer
//     rows through a conflict-free XOR swizzle (fp32: row `lane` = its 16 channels; split: row p = the 32 hi channels of
//     pixel row p, row 16 + p = the 32 lo channels), and 4 consecutive lanes then store one buffer row: 64 contiguous
//     bytes of one pixel.
// Chunks that are not 32 full, 16-byte-aligned channels take the direct path.
template <int BN, bool T3 = false, bool DACT = false>
__device__ __forceinline__ void epilogue_tile(const Params& p, const TileCoord& t, const float* acc, int row0, int cog,
                                              const float* __restrict__ bias_s, uint8_t* __restrict__ stage, const int TW,
                                              const int TH) {
  const int lane = threadIdx.x & 31;
  const int hf = lane >> 4;                            // which 16 channels of a 32-channel chunk this lane handles
  const int r = row0 + (lane & 15);                    // this lane's accumulator row
  // accumulator row R -> GEMM-grid pixel (gy, gx) -> output pixel (Y, X) of the out_H x out_W image
  auto map_row = [&](int R, int& Y, int& X) -> bool {
    const int ly = R / TW, gy = t.y0 + ly, gx = t.x0 + (R - ly * TW);
    Y = gy * p.ostep + t.oy;
    X = gx * p.ostep + t.ox;
    return ly < TH && gy < p.H && gx < p.W && Y < p.out_H && X < p.out_W;
  };
  int y, x;                                            // this thread's OUTPUT pixel
  const bool pix_ok = map_row(r, y, x);
  // pixel indices of this thread's output pixel, computed where used (the fp32 accumulator fills most registers)
  auto pix = [&] { return static_cast<size_t>(t.n) * p.out_nstride + static_cast<size_t>(y) * p.out_W + x; };          // fp32 out, residual
  auto opix = [&] { return static_cast<size_t>(t.n) * p.osp_nstride + static_cast<size_t>(y) * p.out_pitch + p.out_lead + x; };  // split outputs
  auto mpix = [&] { return static_cast<size_t>(y) * p.out_W + x; };                                    // bias map
  auto dpix = [&] { return static_cast<size_t>(t.n) * p.dact_nstride + static_cast<size_t>(y) * p.dact_pitch + p.dact_lead + x; };  // dact
  const int co_end = (t.g + 1) * cog;               // exclusive end of this group's output channels
  const bool vec_ok = (p.Cout & 3) == 0;            // 16-byte aligned channel groups
  const uint32_t sbase = smem_u32(stage);
#pragma unroll                                      // compile-time fragment indices: acc stays in registers
  for (int c = 0; c < BN / 32; ++c) {
    // ---------------------------------------------------------------- 1 + 2: fragments -> row-wise values
    __syncwarp();                                   // the previous chunk's stores have read the buffer
    const int qa = lane >> 2, qc = (lane & 3) >> 1, qo = (lane & 1) * 8;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * c + jj;                     // columns 8j + 2 (lane % 4) + {0, 1} of rows qa, qa + 8
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
    __syncwarp();                                   // every lane has its values before the buffer is reused
    const int co_chunk = t.co0 + c * 32, co = co_chunk + 16 * hf;
    if (vec_ok && co_chunk + 32 <= co_end) {
      // ------------------------------------------------------------ 3: staged, coalesced stores (warp-uniform branch)
      float f[16];
#pragma unroll
      for (int g4 = 0; g4 < 4; ++g4) {
        const float4 b = *reinterpret_cast<const float4*>(bias_s + co + g4 * 4);
        const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float a = __uint_as_float(v[g4 * 4 + i]) + bb[i];
          f[g4 * 4 + i] = a > 0.f ? a : a * p.slope;
        }
      }
      if (p.residual && pix_ok) {
        const float4* r4 = reinterpret_cast<const float4*>(p.residual + pix() * p.Cout + co);
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          const float4 ra = __ldg(r4 + g4);
          f[g4 * 4] += ra.x; f[g4 * 4 + 1] += ra.y; f[g4 * 4 + 2] += ra.z; f[g4 * 4 + 3] += ra.w;
        }
      }
      if constexpr (T3 || DACT) {
        if (p.dact && pix_ok) {
          const uint4* d4 = reinterpret_cast<const uint4*>(p.dact + dpix() * p.Cout + co);
#pragma unroll
          for (int h8 = 0; h8 < 2; ++h8) {
            const uint4 u = __ldg(d4 + h8);
            const __nv_bfloat16* m = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (!(__bfloat162float(m[i]) > 0.f)) f[h8 * 8 + i] *= p.dact_slope;
          }
        }
      }
      if (p.bias_map && pix_ok) {
        const float4* m4 = reinterpret_cast<const float4*>(p.bias_map + mpix() * p.Cout + co);
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          const float4 ra = __ldg(m4 + g4);
          f[g4 * 4] += ra.x; f[g4 * 4 + 1] += ra.y; f[g4 * 4 + 2] += ra.z; f[g4 * 4 + 3] += ra.w;
        }
      }
      // logical 16-byte chunk cc of buffer row rr sits at physical chunk cc ^ ((rr >> 1) & 3); on the read side lanes
      // 4k..4k+3 fetch the 4 chunks of buffer row jr*8 + k.  Both sides touch 8 distinct bank groups per quarter-warp.
      const int sub = lane & 3, prow = lane >> 2;
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
      if (p.out) {                                  // buffer row lane = its 16 fp32 channels: row rr is accumulator row
                                                    // row0 + rr % 16, channels 16 (rr / 16) .. + 16 of the chunk
#pragma unroll
        for (int cc = 0; cc < 4; ++cc)
          st_chunk(lane, cc, __float_as_uint(f[cc * 4]), __float_as_uint(f[cc * 4 + 1]), __float_as_uint(f[cc * 4 + 2]),
                   __float_as_uint(f[cc * 4 + 3]));
        __syncwarp();
#pragma unroll
        for (int jr = 0; jr < 4; ++jr) {
          const int rr = jr * 8 + prow;
          int yy, xx;
          const bool ok = map_row(row0 + (rr & 15), yy, xx);
          const uint4 u = ld_chunk(rr);
          if (ok)
            *reinterpret_cast<uint4*>(p.out + (static_cast<size_t>(t.n) * p.out_nstride + static_cast<size_t>(yy) * p.out_W + xx) * p.out_cs +
                                      co_chunk + 16 * (rr >> 4) + sub * 4) = u;
        }
        __syncwarp();
      }
      if (p.out_hi) {                               // buffer rows [0, 16): 32 bf16 hi channels per pixel row, [16, 32): lo
        uint32_t hp[8], lp[8];                      // packed bf16 pairs
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const __nv_bfloat162 hb = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
          const float2 hfl = __bfloat1622float2(hb);
          const __nv_bfloat162 lb = __floats2bfloat162_rn(f[2 * i] - hfl.x, f[2 * i + 1] - hfl.y);
          hp[i] = *reinterpret_cast<const uint32_t*>(&hb);
          lp[i] = *reinterpret_cast<const uint32_t*>(&lb);
        }
        const int pr = lane & 15;                   // this lane's pixel row; its 16 channels are chunks 2 hf, 2 hf + 1
        st_chunk(pr, 2 * hf, hp[0], hp[1], hp[2], hp[3]);
        st_chunk(pr, 2 * hf + 1, hp[4], hp[5], hp[6], hp[7]);
        st_chunk(16 + pr, 2 * hf, lp[0], lp[1], lp[2], lp[3]);
        st_chunk(16 + pr, 2 * hf + 1, lp[4], lp[5], lp[6], lp[7]);
        __syncwarp();
#pragma unroll
        for (int jr = 0; jr < 4; ++jr) {
          const int rr = jr * 8 + prow;
          int yy, xx;
          const bool ok = map_row(row0 + (rr & 15), yy, xx);
          const uint4 u = ld_chunk(rr);
          __nv_bfloat16* dst = rr < 16 ? p.out_hi : p.out_lo;
          if (ok)
            *reinterpret_cast<uint4*>(dst + (static_cast<size_t>(t.n) * p.osp_nstride + static_cast<size_t>(yy) * p.out_pitch + p.out_lead + xx) *
                                            p.out_cs + co_chunk + sub * 8) = u;
        }
        __syncwarp();
      }
    } else if (pix_ok && co < co_end) {
#pragma unroll
      for (int g8 = 0; g8 < 2; ++g8) {              // 8 output channels at a time
        const int cb = co + g8 * 8;
        if (vec_ok && cb + 8 <= co_end) {
          float f[8];
          const float4 b0 = *reinterpret_cast<const float4*>(bias_s + cb), b1 = *reinterpret_cast<const float4*>(bias_s + cb + 4);
          const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float a = __uint_as_float(v[g8 * 8 + i]) + bb[i];
            f[i] = a > 0.f ? a : a * p.slope;
          }
          if (p.residual) {
            const float4* r4 = reinterpret_cast<const float4*>(p.residual + pix() * p.Cout + cb);
            const float4 ra = __ldg(r4), rb = __ldg(r4 + 1);
            f[0] += ra.x; f[1] += ra.y; f[2] += ra.z; f[3] += ra.w;
            f[4] += rb.x; f[5] += rb.y; f[6] += rb.z; f[7] += rb.w;
          }
          if constexpr (T3 || DACT) {
            if (p.dact) {
              const uint4 u = __ldg(reinterpret_cast<const uint4*>(p.dact + dpix() * p.Cout + cb));
              const __nv_bfloat16* m = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (!(__bfloat162float(m[i]) > 0.f)) f[i] *= p.dact_slope;
            }
          }
          if (p.bias_map) {
            const float4* r4 = reinterpret_cast<const float4*>(p.bias_map + mpix() * p.Cout + cb);
            const float4 ra = __ldg(r4), rb = __ldg(r4 + 1);
            f[0] += ra.x; f[1] += ra.y; f[2] += ra.z; f[3] += ra.w;
            f[4] += rb.x; f[5] += rb.y; f[6] += rb.z; f[7] += rb.w;
          }
          if (p.out) {
            float4* d4 = reinterpret_cast<float4*>(p.out + pix() * p.out_cs + cb);
            d4[0] = make_float4(f[0], f[1], f[2], f[3]);
            d4[1] = make_float4(f[4], f[5], f[6], f[7]);
          }
          if (p.out_hi) {
            uint32_t hp[4], lp[4];                  // packed bf16 pairs, kept in registers
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const __nv_bfloat162 hb = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
              const float2 hfl = __bfloat1622float2(hb);
              const __nv_bfloat162 lb = __floats2bfloat162_rn(f[2 * i] - hfl.x, f[2 * i + 1] - hfl.y);
              hp[i] = *reinterpret_cast<const uint32_t*>(&hb);
              lp[i] = *reinterpret_cast<const uint32_t*>(&lb);
            }
            *reinterpret_cast<uint4*>(p.out_hi + opix() * p.out_cs + cb) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
            *reinterpret_cast<uint4*>(p.out_lo + opix() * p.out_cs + cb) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
          }
        } else if (cb < co_end) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (cb + i < co_end) {
              float a = __uint_as_float(v[g8 * 8 + i]) + bias_s[cb + i];
              a = a > 0.f ? a : a * p.slope;
              if (p.residual) a += __ldg(p.residual + pix() * p.Cout + cb + i);
              if constexpr (T3 || DACT) {
                if (p.dact && !(__bfloat162float(p.dact[dpix() * p.Cout + cb + i]) > 0.f)) a *= p.dact_slope;
              }
              if (p.bias_map) a += __ldg(p.bias_map + mpix() * p.Cout + cb + i);
              if (p.epi_flags & EPI_TANH) a = tanhf(a);
              if (p.out) {
                if (p.epi_flags & EPI_NCHW)   // thread = pixel: consecutive lanes write consecutive x of one channel plane
                  p.out[((static_cast<size_t>(t.n) * p.Cout + cb + i) * p.out_H + y) * p.out_W + x] = a;
                else
                  p.out[pix() * p.out_cs + cb + i] = a;
              }
              if (p.out_hi) {
                const __nv_bfloat16 hb = __float2bfloat16_rn(a);
                p.out_hi[opix() * p.out_cs + cb + i] = hb;
                p.out_lo[opix() * p.out_cs + cb + i] = __float2bfloat16_rn(a - __bfloat162float(hb));
              }
            }
          }
        }
      }
    }
  }
  // row-gapped split output: the pixel at x == 0 also writes the zero gap in front of its row, the very last pixel
  // the zero tail (once per pixel: only the first-half lane of the first N tile of group 0 does it; Cout % 8 == 0 is
  // checked by the API)
  if (p.out_hi && p.out_lead && pix_ok && t.co0 == 0 && hf == 0) {
    const uint4 z = make_uint4(0, 0, 0, 0);
    if (x == 0) {
      uint4* zh = reinterpret_cast<uint4*>(p.out_hi + (opix() - p.out_lead) * p.Cout);
      uint4* zl = reinterpret_cast<uint4*>(p.out_lo + (opix() - p.out_lead) * p.Cout);
      for (int i = 0; i < p.out_lead * p.Cout / 8; ++i) zh[i] = zl[i] = z;
    }
    if (x == p.out_W - 1 && y == p.out_H - 1 && t.n == p.N - 1) {
      uint4* zh = reinterpret_cast<uint4*>(p.out_hi + (opix() + 1) * p.Cout);
      uint4* zl = reinterpret_cast<uint4*>(p.out_lo + (opix() + 1) * p.Cout);
      for (int i = 0; i < p.out_tail * p.Cout / 8; ++i) zh[i] = zl[i] = z;
    }
  }
}

// T3: 3-D conv over NDHWC sources through 5-D tensor maps {C, W, H, T, B} (see Params::t_out); the 2-D instantiations
// are unchanged.  DACT: 2-D, and the epilogue also applies Params::dact (conv3x3_dact_kernel: the input gradients of
// SPyNet's 7x7 convs); the plain 2-D instantiations compile without that code.
template <int BN, bool T3, bool DACT>
__device__ __forceinline__ void conv3x3_body(const Maps& maps, const Params& p) {
  constexpr int W_TILE = Cfg<BN>::W_TILE, STAGE = Cfg<BN>::STAGE, STAGES = Cfg<BN>::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE);
  uint64_t* empty = full + STAGES;
  float* bias_s = reinterpret_cast<float*>(smem + STAGES * STAGE + 256);
  uint8_t* epi_stage = smem + STAGES * STAGE + 256 + MAX_COUT * 4;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < MAX_COUT; i += blockDim.x) bias_s[i] = (p.bias && i < p.Cout) ? __ldg(p.bias + i) : 0.f;
  const int tiles_y = (p.H + p.tile_h - 1) / p.tile_h, tiles_x = (p.W + p.tile_w - 1) / p.tile_w;
  const int cog = p.Cout / p.groups;
  const int tiles_ng = (cog + BN - 1) / BN;
  const int num_tiles = p.N * tiles_y * tiles_x * p.nphase * p.groups * tiles_ng;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);                           // the 4 warps of the warpgroup that consumed the stage
    }
    fence_barrier_init();
    tma_prefetch_desc(&maps.w_hi);
    tma_prefetch_desc(&maps.w_lo);
    for (int i = 0; i < p.nsrc; ++i) {
      tma_prefetch_desc(&maps.a_hi[i]);
      tma_prefetch_desc(&maps.a_lo[i]);
    }
  }
  __syncthreads();

  if (warp >= EPI_WARPS) {
    // ------------------------------------------------------------------ TMA producer (im2col by coordinates), one ring
    regs_dec<PRODUCER_REGS>();
    if (warp == EPI_WARPS && elect_one()) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord t = decode_tile<BN>(tile, p, tiles_y, tiles_x, tiles_ng);
        int kb = 0;
        // bytes a stage receives: two A boxes of tile_w * tile_h rows x 128 B (rows beyond stay idle) + [Wh | Wl]
        const uint32_t stage_tx = 2u * static_cast<uint32_t>(p.tile_w * p.tile_h) * 128u + 2u * W_TILE;
        if constexpr (T3) {
          const int b = t.n / p.t_out, to = t.n - b * p.t_out;
          if (p.rows_px) {
            // window-packed K over (kt, ky, g): kt frames, ky rows, window g of the kernel row
            for (int k = 0; k < p.kt; ++k) {
              const int ti = to * p.tstride - p.tpad + k;
              for (int ky = 0; ky < p.ks; ++ky) {
                const int yy = t.y0 * p.stride - p.pad + ky;
                for (int g = 0; g < p.rows_g; ++g, ++kb, ++it) {
                  const int stage = it % STAGES;
                  mbar_wait(&empty[stage], ((it / STAGES) & 1) ^ 1);
                  mbar_arrive_expect_tx(&full[stage], stage_tx);
                  const uint32_t s0 = smem_u32(smem + stage * STAGE);
                  const int xi = t.x0 + g * p.rows_px / p.stride;
                  tma_load_5d(s0, &maps.a_hi[0], &full[stage], 0, xi, yy, ti, b);
                  tma_load_5d(s0 + A_TILE, &maps.a_lo[0], &full[stage], 0, xi, yy, ti, b);
                  tma_load_2d(s0 + 2 * A_TILE, &maps.w_hi, &full[stage], kb * BK, t.co0);
                  tma_load_2d(s0 + 2 * A_TILE + W_TILE, &maps.w_lo, &full[stage], kb * BK, t.co0);
                }
              }
            }
            continue;
          }
          // taps of this tile's phase; (y, x) steps by `stride` (the TMA box is traversed with that element stride)
          const int tap0 = p.ph_tap0[t.ph], tap1 = p.ph_tap0[t.ph + 1];
          kb = tap0 * p.chunks[0];
          for (int tap = tap0; tap < tap1; ++tap) {
            const int yy = t.y0 * p.stride + p.tap_dy[tap], xx = t.x0 * p.stride + p.tap_dx[tap], ti = to + p.tap_dt[tap];
            for (int j = 0; j < p.chunks[0]; ++j, ++kb, ++it) {
              const int stage = it % STAGES;
              mbar_wait(&empty[stage], ((it / STAGES) & 1) ^ 1);
              mbar_arrive_expect_tx(&full[stage], stage_tx);
              const uint32_t s0 = smem_u32(smem + stage * STAGE);
              tma_load_5d(s0, &maps.a_hi[0], &full[stage], j * BK, xx, yy, ti, b);
              tma_load_5d(s0 + A_TILE, &maps.a_lo[0], &full[stage], j * BK, xx, yy, ti, b);
              tma_load_2d(s0 + 2 * A_TILE, &maps.w_hi, &full[stage], kb * BK, t.co0);
              tma_load_2d(s0 + 2 * A_TILE + W_TILE, &maps.w_lo, &full[stage], kb * BK, t.co0);
            }
          }
          continue;
        }
        if (p.rows_px) {
          // window-packed K: chunk (ky, g) = pixels [x*stride - pad + g*PX, +PX) x cin of input row y*stride - pad + ky
          for (int ky = 0; ky < p.ks; ++ky) {
            const int yy = t.y0 * p.stride - p.pad + ky;
            for (int g = 0; g < p.rows_g; ++g, ++kb, ++it) {
              const int stage = it % STAGES;
              mbar_wait(&empty[stage], ((it / STAGES) & 1) ^ 1);
              mbar_arrive_expect_tx(&full[stage], stage_tx);
              const uint32_t s0 = smem_u32(smem + stage * STAGE);
              const int xi = t.x0 + g * p.rows_px / p.stride;       // window-start index (row gap = left padding)
              tma_load_4d(s0, &maps.a_hi[0], &full[stage], 0, xi, yy, t.n);
              tma_load_4d(s0 + A_TILE, &maps.a_lo[0], &full[stage], 0, xi, yy, t.n);
              tma_load_2d(s0 + 2 * A_TILE, &maps.w_hi, &full[stage], kb * BK, t.co0);
              tma_load_2d(s0 + 2 * A_TILE + W_TILE, &maps.w_lo, &full[stage], kb * BK, t.co0);
            }
          }
          continue;
        }
        const int tap0 = p.ph_tap0[t.ph], tap1 = p.ph_tap0[t.ph + 1];
        kb = tap0 * p.chunks_total;                      // K blocks of the packed weight are ordered by tap
        for (int tap = tap0; tap < tap1; ++tap) {
          // input coordinate of the tile's first output pixel for this tap (TMA steps by `stride` inside the box)
          const int yy = t.y0 * p.stride + p.tap_dy[tap], xx = t.x0 * p.stride + p.tap_dx[tap];
          for (int s = 0; s < p.nsrc; ++s) {
            const int c_base = t.g * p.cig[s];
            for (int j = 0; j < p.chunks[s]; ++j, ++kb, ++it) {
              const int stage = it % STAGES;
              mbar_wait(&empty[stage], ((it / STAGES) & 1) ^ 1);
              mbar_arrive_expect_tx(&full[stage], stage_tx);
              const uint32_t s0 = smem_u32(smem + stage * STAGE);
              tma_load_4d(s0, &maps.a_hi[s], &full[stage], c_base + j * BK, xx, yy, t.n);
              tma_load_4d(s0 + A_TILE, &maps.a_lo[s], &full[stage], c_base + j * BK, xx, yy, t.n);
              tma_load_2d(s0 + 2 * A_TILE, &maps.w_hi, &full[stage], kb * BK, t.co0);
              tma_load_2d(s0 + 2 * A_TILE + W_TILE, &maps.w_lo, &full[stage], kb * BK, t.co0);
            }
          }
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
    uint8_t* my_stage = epi_stage + warp * EPI_STAGE;
    float acc[BN];                                      // rows [0, 64) of the tile, then rows [64, 128)
    // this CTA's tiles: tile blockIdx.x + i * gridDim.x for i < my_tiles; warpgroup wg takes i = wg, wg + 2, ...
    const int grid = static_cast<int>(gridDim.x);
    const int my_tiles = (num_tiles - static_cast<int>(blockIdx.x) + grid - 1) / grid;
    uint32_t it = 0;                                    // ring position of tile i's first K block
    for (int i = 0; i < my_tiles; ++i) {
      const int tile = static_cast<int>(blockIdx.x) + i * grid;
      // K blocks of this tile: the 9-phase gather conv's phases have different tap counts, so the ring position of a
      // tile is the sum over all earlier tiles of the CTA, including the other warpgroup's
      int num_kb = p.ks * p.rows_g;                     // window-packed K
      if constexpr (T3) num_kb *= p.kt;
      if (!p.rows_px) {
        const int ph = (tile / (tiles_ng * p.groups)) % p.nphase;
        num_kb = (p.ph_tap0[ph + 1] - p.ph_tap0[ph]) * p.chunks_total;
      }
      if ((i & 1) != wg) {
        it += num_kb;
        continue;
      }
      // wait for the turn: the other warpgroup has issued tile i - 1's main loop
      if (i > 0) named_sync(ORDER_BAR + wg, 256);
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
          wgmma_ss<BN, false>(acc + BN / 2, dal + HALF, dwh, (kb | k) != 0);
          wgmma_ss<BN, false>(acc, dah, dwl, 1);
          wgmma_ss<BN, false>(acc + BN / 2, dah + HALF, dwl, 1);
          wgmma_ss<BN, false>(acc, dah, dwh, 1);
          wgmma_ss<BN, false>(acc + BN / 2, dah + HALF, dwh, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();                                  // the previous K block's MMAs are done: release its stage
        if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
      }
      if (i + 1 < my_tiles) named_arrive(ORDER_BAR + (wg ^ 1), 256);   // the other warpgroup may issue tile i + 1
      wgmma_wait<0>();
      if (num_kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
      const TileCoord t = decode_tile<BN>(tile, p, tiles_y, tiles_x, tiles_ng);
      // rows wq*16 and 64 + wq*16 through ONE inlined epilogue: the second half is then moved into the first half's
      // registers.  Two inlined copies spill at BN = 128 (124 bytes at 232 registers); this form spills nothing.
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        epilogue_tile<BN, T3, DACT>(p, t, acc, h * 64 + wq * 16, cog, bias_s, my_stage, p.tile_w, p.tile_h);
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = acc[BN / 2 + j];
      }
    }
  }
}

template <int BN, bool T3>
__global__ void __launch_bounds__(THREADS, 1) conv3x3_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p) {
  conv3x3_body<BN, T3, false>(maps, p);
}

template <int BN>
__global__ void __launch_bounds__(THREADS, 1) conv3x3_dact_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p) {
  conv3x3_body<BN, false, true>(maps, p);
}

// ---------------------------------------------------------------------------------------------------------------------
// HALO variant for the low-Cout, high-resolution 3x3 / stride 1 / pad 1 layers (encoder conv 2, decoder deconv-2 conv, the
// 3-channel output conv: Cout <= 64, groups 1).  There the generic kernel is bound by the L2 -> SM fabric (~6300 B/clk
// chip-wide): every 64-channel chunk of a tile is fetched nine times, once per tap, and the matching weight tile comes
// along every time — 432 KB per 128 x 64 output tile against 3456 MMA cycles.  Here
//  * the tile is 8 x 16 pixels and ONE TMA box {64 ch, 10 x, 18 y} per (chunk, hi | lo) brings its whole halo
//    (23 KB instead of 9 x 16 KB); tap (dy, dx) reads it in place through a wgmma descriptor whose start address is shifted
//    by (dy*10 + dx) pixels of 128 B and whose 8-row-group stride (SBO) is one halo row, 1280 B.  The 128B swizzle is a
//    function of absolute shared-memory address bits, so the shifted start needs no base offset;
//  * all weight tiles of the layer (9 taps x chunks x [Wh | Wl]) are loaded ONCE per persistent CTA and stay in shared
//    memory, so steady-state L2 traffic is the 46 KB halo pair per chunk;
//  * the halo ring holds single (hi or lo) pieces: all Ah MMAs of a chunk (9 taps x 4, against Wh and Wl) are issued
//    from one piece, then all Al MMAs (against Wh) from the next.
constexpr int HTILE_W = 8, HTILE_H = 16, HALO_W = HTILE_W + 2, HALO_H = HTILE_H + 2;
constexpr int HALO_BYTES = HALO_W * HALO_H * BK * 2;     // 23040
constexpr int HALO_SLOT = 23552;                        // rounded up to the 1024-byte swizzle atom
constexpr int HALO_MAX_SLOTS = 6;
constexpr int SMEM_LIMIT = 232448;                      // 227 KB opt-in maximum per CTA
constexpr int HALO_THREADS = (EPI_WARPS + 1) * 32;      // two consumer warpgroups (64 accumulator rows each) + the TMA warp

__host__ __device__ constexpr int halo_w_bytes(int bn, int chunks_total) { return 9 * chunks_total * 2 * bn * BK * 2; }

template <int BN>
__global__ void __launch_bounds__(HALO_THREADS, 1) conv3x3_halo_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p,
                                                                  const int nslots) {
  constexpr int W_TILE = Cfg<BN>::W_TILE;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int w_bytes = halo_w_bytes(BN, p.chunks_total);
  uint8_t* ring = smem + w_bytes;                                   // w_bytes is a multiple of 1024
  uint64_t* a_full = reinterpret_cast<uint64_t*>(ring + nslots * HALO_SLOT);
  uint64_t* a_empty = a_full + HALO_MAX_SLOTS;
  uint64_t* w_full = a_empty + HALO_MAX_SLOTS;
  float* bias_s = reinterpret_cast<float*>(ring + nslots * HALO_SLOT + 256);
  uint8_t* epi_stage = ring + nslots * HALO_SLOT + 256 + MAX_COUT * 4;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < MAX_COUT; i += blockDim.x) bias_s[i] = (p.bias && i < p.Cout) ? __ldg(p.bias + i) : 0.f;
  const int tiles_y = (p.H + HTILE_H - 1) / HTILE_H, tiles_x = (p.W + HTILE_W - 1) / HTILE_W;
  const int num_tiles = p.N * tiles_y * tiles_x;

  if (tid == 0) {
    for (int s = 0; s < nslots; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], EPI_WARPS);
    }
    mbar_init(w_full, 1);
    fence_barrier_init();
    tma_prefetch_desc(&maps.w_hi);
    tma_prefetch_desc(&maps.w_lo);
    for (int i = 0; i < p.nsrc; ++i) {
      tma_prefetch_desc(&maps.a_hi[i]);
      tma_prefetch_desc(&maps.a_lo[i]);
    }
  }
  __syncthreads();

  if (warp == EPI_WARPS) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      // resident weights: slot (tap, chunk) = [Wh (BN rows) | Wl (BN rows)], K column of the packed weight = (tap, chunk)
      mbar_arrive_expect_tx(w_full, static_cast<uint32_t>(w_bytes));
      for (int tap = 0; tap < 9; ++tap)
        for (int c = 0; c < p.chunks_total; ++c) {
          const int kb = tap * p.chunks_total + c;
          const uint32_t dst = smem_u32(smem) + kb * 2 * W_TILE;
          tma_load_2d(dst, &maps.w_hi, w_full, kb * BK, 0);
          tma_load_2d(dst + W_TILE, &maps.w_lo, w_full, kb * BK, 0);
        }
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, n = tile / (tiles_x * tiles_y);
        const int xx = tx * HTILE_W - 1, yy = ty * HTILE_H - 1;
        for (int s = 0; s < p.nsrc; ++s)
          for (int j = 0; j < p.chunks[s]; ++j)
            for (int part = 0; part < 2; ++part, ++it) {
              const int slot = it % nslots;
              mbar_wait(&a_empty[slot], ((it / nslots) & 1) ^ 1);
              mbar_arrive_expect_tx(&a_full[slot], HALO_BYTES);
              tma_load_4d(smem_u32(ring + slot * HALO_SLOT), part ? &maps.a_lo[s] : &maps.a_hi[s], &a_full[slot], j * BK,
                          xx, yy, n);
            }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: wgmma main loop, then the epilogue
    // warpgroup wg owns tile rows [8 wg, 8 wg + 8) = accumulator rows [64 wg, 64 wg + 64): its A operand starts 8 halo
    // rows further
    const int wg = warp >> 2, wq = warp & 3;
    const uint64_t d_a0 = gmma_desc_sw128(smem_u32(ring) + wg * 8 * HALO_W * 128, 16, HALO_W * 128);
    const uint64_t d_w0 = gmma_desc_sw128(smem_u32(smem), 16, 1024);
    uint8_t* my_stage = epi_stage + warp * EPI_STAGE;
    float acc[BN / 2];
    mbar_wait(w_full, 0);
    uint32_t it = 0;
    const uint32_t wstep = static_cast<uint32_t>(p.chunks_total * 2 * W_TILE) >> 4;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      // one chunk = its hi piece, then its lo piece, in straight-line code: a data-dependent branch between the two MMA
      // sequences makes ptxas serialize every wgmma of the kernel.  Taps are fully unrolled so that the halo shift
      // (dy*10 + dx pixels) is an immediate, one running 64-bit add per weight slot.
      for (int chunk = 0; chunk < p.chunks_total; ++chunk) {
        const uint64_t dw0 = d_w0 + ((chunk * 2 * W_TILE) >> 4);
        int slot = it % nslots;
        mbar_wait(&a_full[slot], (it / nslots) & 1);
        uint64_t da = d_a0 + ((slot * HALO_SLOT) >> 4);
        uint64_t dw = dw0;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap, dw += wstep) {
          const uint64_t dat = da + ((((tap / 3) * HALO_W + tap % 3) * 128) >> 4);
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            wgmma_ss<BN, false>(acc, dat + 2 * k, dw + (W_TILE >> 4) + 2 * k, (chunk | tap | k) != 0);   // Ah.Wl
            wgmma_ss<BN, false>(acc, dat + 2 * k, dw + 2 * k, 1);                                         // + Ah.Wh
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                  // the previous chunk's lo piece is done: release its slot
        if (chunk > 0 && lane == 0) mbar_arrive(&a_empty[(it - 1) % nslots]);
        ++it;

        slot = it % nslots;
        mbar_wait(&a_full[slot], (it / nslots) & 1);
        da = d_a0 + ((slot * HALO_SLOT) >> 4);
        dw = dw0;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap, dw += wstep) {
          const uint64_t dat = da + ((((tap / 3) * HALO_W + tap % 3) * 128) >> 4);
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) wgmma_ss<BN, false>(acc, dat + 2 * k, dw + 2 * k, 1);        // + Al.Wh
        }
        wgmma_commit();
        wgmma_wait<1>();                                  // this chunk's hi piece is done: release its slot
        if (lane == 0) mbar_arrive(&a_empty[(it - 1) % nslots]);
        ++it;
      }
      wgmma_wait<0>();
      if (p.chunks_total > 0 && lane == 0) mbar_arrive(&a_empty[(it - 1) % nslots]);
      TileCoord t;
      t.x0 = (tile % tiles_x) * HTILE_W;
      t.y0 = ((tile / tiles_x) % tiles_y) * HTILE_H;
      t.n = tile / (tiles_x * tiles_y);
      t.g = 0;
      t.co0 = 0;
      t.ph = t.oy = t.ox = 0;
      epilogue_tile<BN>(p, t, acc, wg * 64 + wq * 16, p.Cout, bias_s, my_stage, HTILE_W, HTILE_H);
    }
  }
}

// NCHW fp32 (C <= cin channels) -> row-gapped NHWC bf16 (hi, lo) [N][H][lead + W][cin] + tail, zeros in the gaps, the
// tail and channels >= C: the operand layout of the window-packed conv.  One thread per (row pixel incl. gap, n*H+y).
__global__ void __launch_bounds__(256) pack_rows_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                                                        __nv_bfloat16* __restrict__ lo, int N, int C, int H, int W, int cin,
                                                        int lead, int pitch, int tail) {
  const long long total = static_cast<long long>(N) * H * pitch + tail;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long row = i / pitch;
  const int xp = static_cast<int>(i - row * pitch) - lead;
  const bool inside = row < static_cast<long long>(N) * H && xp >= 0 && xp < W;
  const long long n = row / H;
  const int y = static_cast<int>(row - n * H);
  for (int c0 = 0; c0 < cin; c0 += 4) {          // cin is a multiple of 4: 8-byte stores
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      f[j] = (inside && c0 + j < C) ? __ldg(x + ((n * C + c0 + j) * H + y) * static_cast<long long>(W) + xp) : 0.f;
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(f[0], f[1]), h1 = __floats2bfloat162_rn(f[2], f[3]);
    const float2 g0 = __bfloat1622float2(h0), g1 = __bfloat1622float2(h1);
    const __nv_bfloat162 l0 = __floats2bfloat162_rn(f[0] - g0.x, f[1] - g0.y), l1 = __floats2bfloat162_rn(f[2] - g1.x, f[3] - g1.y);
    *reinterpret_cast<uint2*>(hi + i * cin + c0) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
    *reinterpret_cast<uint2*>(lo + i * cin + c0) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side shared by the generic kernel's three launchers: launch_conv3x3 (2-D and gather convs), launch_conv3d (I3D)
// and launch_dis_conv (the discriminator).

// Tile shape of an h x w GEMM grid.  Images smaller than a 16 x 8 tile (SPyNet's coarse pyramid levels: 2x4, 4x8 pixels)
// take a tile of their own size: the A boxes shrink from 16 KB to 1-4 KB per K block, and these few-CTA launches are
// bound by the per-SM L2 port.  Otherwise, unless `search` is off (a row-gapped source keeps 16 x 8), the
// tile_w x tile_h <= 128 box that covers the image with the FEWEST tiles: at 60 x 108 (every propagation / encoder conv
// of a 432x240 clip) 12 x 10 tiles the image exactly with 54 tiles where 16 x 8 needs 56 — at 8 clips that is 432
// instead of 448 tiles.  The candidates have tw <= 32 and th <= 16, and every launcher that searches runs at stride 1
// or 2, so a source box (tile * stride elements per axis) stays within TMA's 256 without a check here.
static void pick_tile(int h, int w, bool search, int& tile_w, int& tile_h) {
  tile_w = w < TILE_W ? w : TILE_W;
  tile_h = h < TILE_H ? h : TILE_H;
  if (w < TILE_W || h < TILE_H || !search) return;
  long long best = static_cast<long long>((h + TILE_H - 1) / TILE_H) * ((w + TILE_W - 1) / TILE_W);
  for (int tw = 32; tw >= 8; --tw) {                        // ties go to the wider tile (longer contiguous TMA rows)
    const int th = BM / tw;
    if (th < 4 || th > h || tw > w) continue;
    const long long cnt = static_cast<long long>((h + th - 1) / th) * ((w + tw - 1) / tw);
    if (cnt < best) {
      best = cnt;
      tile_w = tw;
      tile_h = th;
    }
  }
}

// N tile (see Cfg) for `cog` output channels per group, the same rule for every launcher.  The N tile only splits the
// output channels: no element's K summation depends on it, so a layer computes the same bits at any BN.  (The
// discriminator's layers have 8-128 channels but never 96.)
static int pick_bn(int cog) { return cog <= 32 ? 32 : cog <= 64 ? 64 : cog == 96 ? 96 : 128; }

// the hi and lo maps of one bf16 operand pair: the same geometry over two buffers
static int encode_pair(CUtensorMap& map_hi, CUtensorMap& map_lo, const void* hi, const void* lo, int rank,
                       const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr,
                       const char* what) {
  const int e = encode_tmap(&map_hi, hi, rank, dims, strides, box, estr, what);
  return e ? e : encode_tmap(&map_lo, lo, rank, dims, strides, box, estr, what);
}

// weights [Cout][kpad] bf16 (hi, lo), K blocks in the order the producer walks them: one {64, BN} box per K block
static int encode_weights(Maps& maps, const void* w_hi, const void* w_lo, int kpad, int cout, int bn, const char* what) {
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(kpad), static_cast<cuuint64_t>(cout)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(kpad) * 2};
  const cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(bn)};
  const cuuint32_t estr[2] = {1, 1};
  return encode_pair(maps.w_hi, maps.w_lo, w_hi, w_lo, 2, dims, strides, box, estr, what);
}

// one instantiation, its shared-memory size set once per device
template <int BN, bool T3, bool DACT>
static int launch_bn(const Maps& maps, const Params& p, int grid, cudaStream_t stream) {
  const auto kern = [] {
    if constexpr (DACT) return conv3x3_dact_kernel<BN>;
    else return conv3x3_kernel<BN, T3>;
  }();
  static DeviceOnce configured;
  if (const int e = configure_once(configured, Cfg<BN>::SMEM, kern)) return e;
  kern<<<grid, THREADS, Cfg<BN>::SMEM, stream>>>(maps, p);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// The launchers' common tail: count p's tiles over n images as the kernel does, size the persistent grid and launch the
// instantiation for bn.
template <bool T3, bool DACT = false>
static int launch_tiles(const Maps& maps, const Params& p, long long n, int bn, const char* who, cudaStream_t stream) {
  const long long tiles = n * ((p.H + p.tile_h - 1) / p.tile_h) * ((p.W + p.tile_w - 1) / p.tile_w) * p.nphase * p.groups *
                          ((p.Cout / p.groups + bn - 1) / bn);
  if (tiles == 0) return 0;
  if (tiles > 0x7FFFFFFFLL) {
    set_error("%s: too many tiles", who);
    return -2;
  }
  const int grid = tiles < num_sms() ? static_cast<int>(tiles) : num_sms();
  switch (bn) {
    case 32: return launch_bn<32, T3, DACT>(maps, p, grid, stream);
    case 64: return launch_bn<64, T3, DACT>(maps, p, grid, stream);
    case 96: return launch_bn<96, T3, DACT>(maps, p, grid, stream);
    default: return launch_bn<128, T3, DACT>(maps, p, grid, stream);
  }
}

}  // namespace conv

int conv_rows_tail(int lead, int channels) { return lead + (conv::BK + channels - 1) / channels; }

// pixels per row of the row-gapped layout: lead + W, rounded up so that a row is a multiple of 16 bytes (TMA stride
// rule; only matters for 4 channels); the extra pixel, if any, sits at the END of the row and is zero as well
int conv_rows_pitch(int w, int lead, int channels) {
  const int unit = channels >= 8 ? 1 : 8 / channels;
  return (w + lead + unit - 1) / unit * unit;
}

int launch_pack_rows(const float* x, void* hi, void* lo, int n, int c, int h, int w, int cin, int lead,
                     cudaStream_t stream) {
  const int pitch = conv_rows_pitch(w, lead, cin);
  const long long total = static_cast<long long>(n) * h * pitch + conv_rows_tail(lead, cin);
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  conv::pack_rows_kernel<<<blocks, 256, 0, stream>>>(x, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), n, c,
                                                     h, w, cin, lead, pitch, conv_rows_tail(lead, cin));
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_conv3x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                   const void* w_hi, const void* w_lo, const float* bias, const float* residual, float* out,
                   void* out_hi, void* out_lo, int n, int h_in, int w_in, int cout, int groups, float slope, int ks,
                   int stride, int pad, int in_rows, int out_lead, cudaStream_t stream, const ConvGeom* geom, int epi_flags,
                   const void* dact, int dact_lead, float dact_slope) {
  using namespace conv;
  if (epi_flags && ((cout & 3) == 0 || out_hi || residual || geom)) {
    set_error("conv: tanh / NCHW epilogues are implemented for the element-wise store path (Cout %% 4 != 0, fp32 output only)");
    return -2;
  }
  if (dact && (cout % 8 || (geom && geom->out_nstride > 0))) {
    set_error("conv: the ReLU-derivative epilogue needs Cout %% 8 == 0 and a dense output");
    return -2;
  }
  // GEMM grid = output size of the plain conv, or what the generalised geometry says
  const int h = geom ? geom->grid_h : (h_in + 2 * pad - ks) / stride + 1;
  const int w = geom ? geom->grid_w : (w_in + 2 * pad - ks) / stride + 1;
  int tile_w = geom ? geom->tile_w : 0, tile_h = geom ? geom->tile_h : 0;
  if (!geom) pick_tile(h, w, !in_rows, tile_w, tile_h);
  const int ntaps = geom ? geom->ntaps : ks * ks;
  if (ntaps < 1 || ntaps > 64 || tile_w < 1 || tile_h < 1 || tile_w * tile_h > BM || tile_w * stride > 256 ||
      tile_h * stride > 256 || (geom && (geom->nphase < 1 || geom->nphase > 9 || geom->ostep < 1))) {
    set_error("conv: unsupported geometry (taps=%d tile=%dx%d stride=%d)", ntaps, tile_w, tile_h, stride);
    return -2;
  }
  if (cout > MAX_COUT) {
    set_error("conv3x3: at most %d output channels (the bias is staged in shared memory), got %d", MAX_COUT, cout);
    return -2;
  }
  const int cog = cout / groups;
  int bn = pick_bn(cog);
  // few tiles (single-clip propagation steps: 51 pixel tiles): halve the N tile so that twice as many SMs work
  if (bn == 128 && cog % 64 == 0 && !in_rows) {
    const long long t128 = static_cast<long long>(n) * ((h + tile_h - 1) / tile_h) * ((w + tile_w - 1) / tile_w) * groups *
                           ((cog + 127) / 128) * (geom ? geom->nphase : 1);
    if (2 * t128 <= num_sms()) bn = 64;
  }
  Maps maps;
  Params p;
  memset(&p, 0, sizeof(p));
  p.N = n; p.H = h; p.W = w; p.Cout = cout; p.groups = groups; p.nsrc = nsrc;
  p.ks = ks; p.stride = stride; p.pad = pad;
  p.slope = slope; p.bias = bias; p.residual = residual; p.out = out; p.epi_flags = epi_flags;
  p.out_cs = cout;
  p.out_hi = static_cast<__nv_bfloat16*>(out_hi); p.out_lo = static_cast<__nv_bfloat16*>(out_lo);
  p.out_lead = out_lead;
  p.tile_w = tile_w; p.tile_h = tile_h;
  p.dact = static_cast<const __nv_bfloat16*>(dact); p.dact_lead = dact_lead; p.dact_slope = dact_slope;
  if (geom) {
    p.nphase = geom->nphase; p.ostep = geom->ostep; p.out_H = geom->out_h; p.out_W = geom->out_w;
    p.bias_map = geom->bias_map;
    for (int i = 0; i < ntaps; ++i) { p.tap_dy[i] = geom->tap_dy[i]; p.tap_dx[i] = geom->tap_dx[i]; }
    for (int i = 0; i < geom->nphase; ++i) { p.ph_tap0[i] = geom->ph_tap0[i]; p.ph_oy[i] = geom->ph_oy[i]; p.ph_ox[i] = geom->ph_ox[i]; }
    p.ph_tap0[geom->nphase] = geom->ph_tap0[geom->nphase];
  } else {
    p.nphase = 1; p.ostep = 1; p.out_H = h; p.out_W = w;
    for (int i = 0; i < ntaps; ++i) { p.tap_dy[i] = static_cast<int8_t>(i / ks - pad); p.tap_dx[i] = static_cast<int8_t>(i % ks - pad); }
    p.ph_tap0[1] = static_cast<uint8_t>(ntaps);
  }
  p.out_pitch = conv_rows_pitch(p.out_W, out_lead, cout);   // == out_W + out_lead: split outputs have >= 8 channels
  p.out_nstride = static_cast<long long>(p.out_H) * p.out_W;
  p.osp_nstride = static_cast<long long>(p.out_H) * p.out_pitch;
  if (geom && geom->out_nstride > 0) {                       // batch-strided output (a frame slice of a (b, t, h, w, c) buffer)
    if (out_lead || geom->out_nstride < p.out_nstride) {
      set_error("conv: a batch-strided output needs a dense row layout and a stride >= out_h * out_w pixels");
      return -2;
    }
    p.out_nstride = p.osp_nstride = geom->out_nstride;
  }
  p.out_tail = out_lead ? conv_rows_tail(out_lead, cout) : 0;
  p.dact_pitch = dact_lead ? conv_rows_pitch(p.out_W, dact_lead, cout) : p.out_W;
  p.dact_nstride = static_cast<long long>(p.out_H) * p.dact_pitch;
  long long src_nstride[MAX_SRC];                            // pixels between consecutive images of each dense source
  if (in_rows) {
    p.rows_px = BK / src_channels[0];
    p.rows_g = (ks + p.rows_px - 1) / p.rows_px;
    p.cig[0] = src_channels[0];
    p.chunks[0] = p.chunks_total = 1;
  } else {
    for (int i = 0; i < nsrc; ++i) {
      p.cig[i] = src_channels[i] / groups;
      p.chunks[i] = (p.cig[i] + BK - 1) / BK;
      p.chunks_total += p.chunks[i];
      src_nstride[i] = static_cast<long long>(h_in) * w_in;
      if (geom && geom->src_nstride && geom->src_nstride[i] > 0) {
        if (geom->src_nstride[i] < src_nstride[i]) {
          set_error("conv: source %d batch stride %lld is smaller than one image (%lld pixels)", i, geom->src_nstride[i],
                    src_nstride[i]);
          return -2;
        }
        src_nstride[i] = geom->src_nstride[i];
      }
    }
  }
  // HALO variant (see conv3x3_halo_kernel): dense 3x3 / s1 / p1 layers with <= 64 output channels whose weights fit
  // in shared memory next to >= 3 halo slots.  Every other shape runs on the generic kernel.
  int halo_slots = 0;
  if (!geom && !in_rows && !dact && ks == 3 && stride == 1 && pad == 1 && groups == 1 && cout <= 64) {
    const int room = SMEM_LIMIT - 1024 - 256 - MAX_COUT * 4 - halo_w_bytes(bn, p.chunks_total) - EPI_WARPS * EPI_STAGE;
    if (room >= 3 * HALO_SLOT) halo_slots = room / HALO_SLOT < HALO_MAX_SLOTS ? room / HALO_SLOT : HALO_MAX_SLOTS;
  }
  if (in_rows) {
    // ONE row-gapped source [N][H][w_in + pad][cin] (+ tail): dimension 1 steps by `stride` pixels, dimension 0 spans
    // 64 elements = 64/cin pixels (overlapping windows; validated by tools/tma_window_probe.cu)
    const int cin = src_channels[0], pitch = conv_rows_pitch(w_in, pad, cin);
    const cuuint64_t dims[4] = {BK, static_cast<cuuint64_t>((pitch + stride - 1) / stride), static_cast<cuuint64_t>(h_in),
                                static_cast<cuuint64_t>(n)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(stride) * cin * 2, static_cast<cuuint64_t>(pitch) * cin * 2,
                                   static_cast<cuuint64_t>(h_in) * pitch * cin * 2};
    const cuuint32_t box[4] = {BK, static_cast<cuuint32_t>(tile_w), static_cast<cuuint32_t>(tile_h * stride), 1};
    const cuuint32_t estr[4] = {1, 1, static_cast<cuuint32_t>(stride), 1};
    if (const int e = encode_pair(maps.a_hi[0], maps.a_lo[0], src_hi[0], src_lo[0], 4, dims, strides, box, estr,
                                  "conv2d row-gapped source"))
      return e;
  }
  const cuuint32_t estr4[4] = {1, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1};
  for (int i = 0; i < (in_rows ? 0 : nsrc); ++i) {
    const int c = src_channels[i];
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(c), static_cast<cuuint64_t>(w_in),
                                static_cast<cuuint64_t>(h_in), static_cast<cuuint64_t>(n)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(c) * 2, static_cast<cuuint64_t>(w_in) * c * 2,
                                   static_cast<cuuint64_t>(src_nstride[i]) * c * 2};
    // the box spans TILE*stride input elements and is traversed with elementStrides = stride: TILE elements land
    const cuuint32_t box[4] = {BK, static_cast<cuuint32_t>(halo_slots ? HALO_W : tile_w * stride),
                               static_cast<cuuint32_t>(halo_slots ? HALO_H : tile_h * stride), 1};
    if (const int e = encode_pair(maps.a_hi[i], maps.a_lo[i], src_hi[i], src_lo[i], 4, dims, strides, box, estr4,
                                  "conv2d source"))
      return e;
  }
  const int kpad = (in_rows ? ks * p.rows_g : ntaps * p.chunks_total) * BK;
  if (const int e = encode_weights(maps, w_hi, w_lo, kpad, cout, bn, "conv3x3 weight")) return e;
  if (halo_slots) {
    static DeviceOnce halo_configured;
    if (const int e = configure_once(halo_configured, SMEM_LIMIT, conv3x3_halo_kernel<64>, conv3x3_halo_kernel<32>)) return e;
    const long long htiles = static_cast<long long>(n) * ((h + HTILE_H - 1) / HTILE_H) * ((w + HTILE_W - 1) / HTILE_W);
    if (htiles == 0) return 0;
    if (htiles > 0x7FFFFFFFLL) {
      set_error("conv3x3: too many tiles");
      return -2;
    }
    const int hgrid = htiles < num_sms() ? static_cast<int>(htiles) : num_sms();
    const int hsmem = 1024 + halo_w_bytes(bn, p.chunks_total) + halo_slots * HALO_SLOT + 256 + MAX_COUT * 4 + EPI_WARPS * EPI_STAGE;
    if (bn == 32)
      conv3x3_halo_kernel<32><<<hgrid, HALO_THREADS, hsmem, stream>>>(maps, p, halo_slots);
    else
      conv3x3_halo_kernel<64><<<hgrid, HALO_THREADS, hsmem, stream>>>(maps, p, halo_slots);
    count_launch();
    return static_cast<int>(cudaGetLastError());
  }
  return dact ? launch_tiles<false, true>(maps, p, n, bn, "conv3x3", stream)
              : launch_tiles<false>(maps, p, n, bn, "conv3x3", stream);
}


// 3-D conv (I3D's Unit3D, see i3d.cu): the generic kernel's T3 instantiation.  Dense: one NDHWC source [b][t][h][w][cin]
// (cin % 8 == 0), ks^3 taps, stride 1, per-axis zero padding pad = {t_f, t_b, h_f, h_b, w_f, w_b}.  Window-packed
// (in_rows = lead > 0): the stem's row-gapped source [b][t][h][pitch][4] whose rows have `lead` zero pixels in front,
// stride 2 on every axis.  Outputs [b][t_o][h_o][w_o][out_cs] with this conv's channels at the pointers given.
int launch_conv3d(const void* src_hi, const void* src_lo, int cin, int in_rows, const void* w_hi, const void* w_lo,
                  const float* bias, float* out, void* out_hi, void* out_lo, int out_cs, int b, int t_in, int h_in,
                  int w_in, int cout, int ks, int stride, const int* pad, float slope, cudaStream_t stream) {
  using namespace conv;
  const int t_o = (t_in + pad[0] + pad[1] - ks) / stride + 1;
  const int h = (h_in + pad[2] + pad[3] - ks) / stride + 1;
  const int w = (w_in + pad[4] + pad[5] - ks) / stride + 1;
  int tile_w, tile_h;
  pick_tile(h, w, !in_rows, tile_w, tile_h);
  // the N tile depends on cout alone (no halving for few tiles, unlike launch_conv3x3), so a video's result does not
  // depend on the batch it is computed in
  const int bn = pick_bn(cout);
  const long long n_img = static_cast<long long>(b) * t_o;
  Maps maps;
  Params p;
  memset(&p, 0, sizeof(p));
  p.N = static_cast<int>(n_img); p.H = h; p.W = w; p.Cout = cout; p.groups = 1; p.nsrc = 1;
  p.ks = ks; p.stride = stride; p.pad = pad[2];
  p.t_out = t_o; p.kt = ks; p.tstride = stride; p.tpad = pad[0];
  p.slope = slope; p.bias = bias; p.out = out; p.out_cs = out_cs;
  p.out_hi = static_cast<__nv_bfloat16*>(out_hi); p.out_lo = static_cast<__nv_bfloat16*>(out_lo);
  p.tile_w = tile_w; p.tile_h = tile_h;
  p.nphase = 1; p.ostep = 1; p.out_H = h; p.out_W = w;
  p.out_pitch = w;
  p.out_nstride = p.osp_nstride = static_cast<long long>(h) * w;
  const int ntaps = in_rows ? 1 : ks * ks * ks;
  for (int i = 0; i < ntaps; ++i) {
    p.tap_dt[i] = static_cast<int8_t>(i / (ks * ks) - pad[0]);
    p.tap_dy[i] = static_cast<int8_t>((i / ks) % ks - pad[2]);
    p.tap_dx[i] = static_cast<int8_t>(i % ks - pad[4]);
  }
  p.ph_tap0[0] = 0; p.ph_tap0[1] = static_cast<uint8_t>(ntaps);
  int kpad;
  if (in_rows) {
    // 4-channel rows, dimension 1 steps by 2 pixels (16 B) and dimension 0 spans the 16-pixel window; the base is moved
    // by lead - w_f pixels (even, so 16-byte aligned) so that window xi starts at input column 2 xi - w_f
    const int lead = in_rows, pitch = conv_rows_pitch(w_in, lead, 4);
    p.rows_px = BK / 4;
    p.rows_g = (ks + p.rows_px - 1) / p.rows_px;
    p.cig[0] = 4; p.chunks[0] = 1; p.chunks_total = 1;
    const cuuint64_t dims[5] = {BK, static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h_in), static_cast<cuuint64_t>(t_in),
                                static_cast<cuuint64_t>(b)};
    const cuuint64_t strides[4] = {16, static_cast<cuuint64_t>(pitch) * 8, static_cast<cuuint64_t>(h_in) * pitch * 8,
                                   static_cast<cuuint64_t>(t_in) * h_in * pitch * 8};
    const cuuint32_t box[5] = {BK, static_cast<cuuint32_t>(tile_w), static_cast<cuuint32_t>(tile_h * stride), 1, 1};
    const cuuint32_t estr[5] = {1, 1, static_cast<cuuint32_t>(stride), 1, 1};
    const int shift = (lead - pad[4]) * 4;
    if (const int e = encode_pair(maps.a_hi[0], maps.a_lo[0], static_cast<const __nv_bfloat16*>(src_hi) + shift,
                                  static_cast<const __nv_bfloat16*>(src_lo) + shift, 5, dims, strides, box, estr,
                                  "conv3d row-gapped source"))
      return e;
    kpad = ks * ks * p.rows_g * BK;
  } else {
    p.cig[0] = cin; p.chunks[0] = (cin + BK - 1) / BK; p.chunks_total = p.chunks[0];
    const cuuint64_t dims[5] = {static_cast<cuuint64_t>(cin), static_cast<cuuint64_t>(w_in), static_cast<cuuint64_t>(h_in),
                                static_cast<cuuint64_t>(t_in), static_cast<cuuint64_t>(b)};
    const cuuint64_t strides[4] = {static_cast<cuuint64_t>(cin) * 2, static_cast<cuuint64_t>(w_in) * cin * 2,
                                   static_cast<cuuint64_t>(h_in) * w_in * cin * 2,
                                   static_cast<cuuint64_t>(t_in) * h_in * w_in * cin * 2};
    const cuuint32_t box[5] = {BK, static_cast<cuuint32_t>(tile_w), static_cast<cuuint32_t>(tile_h), 1, 1};
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (const int e = encode_pair(maps.a_hi[0], maps.a_lo[0], src_hi, src_lo, 5, dims, strides, box, estr, "conv3d source"))
      return e;
    kpad = ntaps * p.chunks_total * BK;
  }
  if (const int e = encode_weights(maps, w_hi, w_lo, kpad, cout, bn, "conv3d weight")) return e;
  return launch_tiles<true>(maps, p, n_img, bn, "conv3d", stream);
}

// Temporal PatchGAN discriminator layers (Conv3d 3x5x5, stride (1, 2, 2), padding (1, pad, pad)): the T3 kernel with a
// 75-tap table.  One NDHWC source [b][t][h_src][w_src][cin] (cin % 8 == 0; channels past the weight's are ignored).
//  * forward (transposed = 0): out[b][t][h_out][w_out][cout], h_out = (h_src + 2 pad - 5) / 2 + 1; the source boxes are
//    traversed with element stride 2 in y and x.  Tap (kt, ky, kx) reads frame t + kt - 1, row 2y + ky - pad, column
//    2x + kx - pad; weight [cout][75 taps in (kt, ky, kx) order][ceil(cin / 64) * 64].
//  * input gradient (transposed = 1): the source is dY of the forward conv and the output dX [b][t][h_out][w_out][cout]
//    (h_out, w_out = the forward's input size).  Output pixel (2gy + oy, 2gx + ox) is phase ph = 2 oy + ox; it gathers
//    the taps with ky = oy + pad (mod 2), kx = ox + pad (mod 2), reading dY at (t + 1 - kt, gy + (oy + pad - ky) / 2,
//    gx + (ox + pad - kx) / 2) with stride 1.  Taps are listed phase by phase, each phase in (kt, ky, kx) order, and
//    the weight [cout][75][ceil(cin / 64) * 64] follows that order.  Rows the forward never read get 0.
// `dact` (or null): the epilogue multiplies by LeakyReLU(dact_slope)'s derivative at that saved activation.
int launch_dis_conv(const void* src_hi, const void* src_lo, int cin, const void* w_hi, const void* w_lo, const float* bias,
                    float* out, void* out_hi, void* out_lo, int b, int t, int h_src, int w_src, int h_out, int w_out,
                    int cout, int pad, int transposed, float slope, const void* dact, float dact_slope, cudaStream_t stream) {
  using namespace conv;
  constexpr int KT = 3, KS = 5;
  const int stride = transposed ? 1 : 2;
  const int h = transposed ? (h_out + 1) / 2 : h_out, w = transposed ? (w_out + 1) / 2 : w_out;   // GEMM grid per phase
  int tile_w, tile_h;
  pick_tile(h, w, true, tile_w, tile_h);
  const int bn = pick_bn(cout);
  const long long n_img = static_cast<long long>(b) * t;
  Maps maps;
  Params p;
  memset(&p, 0, sizeof(p));
  p.N = static_cast<int>(n_img); p.H = h; p.W = w; p.Cout = cout; p.groups = 1; p.nsrc = 1;
  p.ks = KS; p.stride = stride; p.pad = pad;
  p.t_out = t; p.kt = KT; p.tstride = 1; p.tpad = 1;
  p.slope = slope; p.bias = bias; p.out = out; p.out_cs = cout;
  p.out_hi = static_cast<__nv_bfloat16*>(out_hi); p.out_lo = static_cast<__nv_bfloat16*>(out_lo);
  p.dact = static_cast<const __nv_bfloat16*>(dact); p.dact_slope = dact_slope;
  p.dact_pitch = w_out; p.dact_lead = 0; p.dact_nstride = static_cast<long long>(h_out) * w_out;
  p.tile_w = tile_w; p.tile_h = tile_h;
  p.out_H = h_out; p.out_W = w_out; p.out_pitch = w_out;
  p.out_nstride = p.osp_nstride = static_cast<long long>(h_out) * w_out;
  int ntaps = 0;
  if (!transposed) {
    p.nphase = 1; p.ostep = 1;
    for (int kt = 0; kt < KT; ++kt)
      for (int ky = 0; ky < KS; ++ky)
        for (int kx = 0; kx < KS; ++kx, ++ntaps) {
          p.tap_dt[ntaps] = static_cast<int8_t>(kt - 1);
          p.tap_dy[ntaps] = static_cast<int8_t>(ky - pad);
          p.tap_dx[ntaps] = static_cast<int8_t>(kx - pad);
        }
    p.ph_tap0[0] = 0;
  } else {
    p.nphase = 4; p.ostep = 2;
    for (int ph = 0; ph < 4; ++ph) {
      const int oy = ph >> 1, ox = ph & 1;
      p.ph_tap0[ph] = static_cast<uint8_t>(ntaps); p.ph_oy[ph] = static_cast<uint8_t>(oy); p.ph_ox[ph] = static_cast<uint8_t>(ox);
      for (int kt = 0; kt < KT; ++kt)
        for (int ky = 0; ky < KS; ++ky)
          for (int kx = 0; kx < KS; ++kx) {
            if (((oy + pad - ky) & 1) || ((ox + pad - kx) & 1)) continue;
            p.tap_dt[ntaps] = static_cast<int8_t>(1 - kt);
            p.tap_dy[ntaps] = static_cast<int8_t>((oy + pad - ky) / 2);
            p.tap_dx[ntaps] = static_cast<int8_t>((ox + pad - kx) / 2);
            ++ntaps;
          }
    }
  }
  p.ph_tap0[p.nphase] = static_cast<uint8_t>(ntaps);
  p.cig[0] = cin; p.chunks[0] = (cin + BK - 1) / BK; p.chunks_total = p.chunks[0];
  const cuuint64_t dims[5] = {static_cast<cuuint64_t>(cin), static_cast<cuuint64_t>(w_src), static_cast<cuuint64_t>(h_src),
                              static_cast<cuuint64_t>(t), static_cast<cuuint64_t>(b)};
  const cuuint64_t strides[4] = {static_cast<cuuint64_t>(cin) * 2, static_cast<cuuint64_t>(w_src) * cin * 2,
                                 static_cast<cuuint64_t>(h_src) * w_src * cin * 2,
                                 static_cast<cuuint64_t>(t) * h_src * w_src * cin * 2};
  const cuuint32_t box[5] = {BK, static_cast<cuuint32_t>(tile_w * stride), static_cast<cuuint32_t>(tile_h * stride), 1, 1};
  const cuuint32_t estr[5] = {1, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1, 1};
  if (const int e = encode_pair(maps.a_hi[0], maps.a_lo[0], src_hi, src_lo, 5, dims, strides, box, estr, "dis_conv source"))
    return e;
  if (const int e = encode_weights(maps, w_hi, w_lo, ntaps * p.chunks_total * BK, cout, bn, "dis_conv weight")) return e;
  return launch_tiles<true>(maps, p, n_img, bn, "dis_conv", stream);
}

// Input gradient of a k x k conv (2-D, see include/e2fgvi_b200.h e2f_conv_dgrad_bf16x3) on launch_conv3x3's kernel: dY
// is the source, dX [n][h_in][w_in][cin] the output.
//  * stride 1, pad k / 2: a plain conv of dY with the rotated, in / out-swapped weight (groups as the forward's);
//  * k = 3, stride 2, pad 1: four output phases (y % 2, x % 2).  Phase ph = 2 oy + ox lists the taps with ky = oy + 1 and
//    kx = ox + 1 (mod 2) in increasing (ky, kx) order — 1, 2, 2 and 4 taps — and tap (ky, kx) reads dY at (gy + (oy + 1 -
//    ky) / 2, gx + (ox + 1 - kx) / 2) for output pixel (2 gy + oy, 2 gx + ox); the weight lists phase 0's taps, then
//    phase 1's, ... with the forward's (unrotated) values.
int launch_conv_dgrad(const void* dy_hi, const void* dy_lo, int dy_c, int dy_lead, const void* w_hi, const void* w_lo,
                      const void* act, const float* residual, float* dx, void* dx_hi, void* dx_lo, int n, int h_in,
                      int w_in, int cin, int groups, int ks, int stride, cudaStream_t stream) {
  using namespace conv;
  const void* srch[1] = {dy_hi};
  const void* srcl[1] = {dy_lo};
  const int ch[1] = {dy_c};
  if (stride == 1)
    return launch_conv3x3(1, srch, srcl, ch, w_hi, w_lo, nullptr, residual, dx, dx_hi, dx_lo, n, h_in, w_in, cin, groups,
                          1.f, ks, 1, ks / 2, dy_lead ? 1 : 0, 0, stream, nullptr, 0, act, 0, 0.2f);
  int8_t dy[9], dxo[9];
  uint8_t tap0[5], oy[4], ox[4];
  int nt = 0;
  for (int ph = 0; ph < 4; ++ph) {
    oy[ph] = static_cast<uint8_t>(ph >> 1);
    ox[ph] = static_cast<uint8_t>(ph & 1);
    tap0[ph] = static_cast<uint8_t>(nt);
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        if (((oy[ph] + 1 - ky) & 1) || ((ox[ph] + 1 - kx) & 1)) continue;
        dy[nt] = static_cast<int8_t>((oy[ph] + 1 - ky) / 2);
        dxo[nt] = static_cast<int8_t>((ox[ph] + 1 - kx) / 2);
        ++nt;
      }
  }
  tap0[4] = static_cast<uint8_t>(nt);
  ConvGeom g;
  memset(&g, 0, sizeof(g));
  g.grid_h = (h_in + 1) / 2;
  g.grid_w = (w_in + 1) / 2;
  g.out_h = h_in;
  g.out_w = w_in;
  pick_tile(g.grid_h, g.grid_w, true, g.tile_w, g.tile_h);
  g.ntaps = nt; g.nphase = 4; g.ostep = 2;
  g.tap_dy = dy; g.tap_dx = dxo; g.ph_tap0 = tap0; g.ph_oy = oy; g.ph_ox = ox;
  const int h_o = (h_in - 1) / 2 + 1, w_o = (w_in - 1) / 2 + 1;
  return launch_conv3x3(1, srch, srcl, ch, w_hi, w_lo, nullptr, residual, dx, dx_hi, dx_lo, n, h_o, w_o, cin, groups, 1.f,
                        3, 1, 0, 0, 0, stream, &g, 0, act, 0, 0.2f);
}

}  // namespace e2f
