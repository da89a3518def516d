// Token <-> image transforms of the T2T path ("soft split" / "soft composition" / fusion feed-forward):
//   t2t_unfold : img [BT][C][H][W] -> tokens [BT][L][C*k*k]   == F.unfold(k, stride, pad).permute(0,2,1)
//                (tfocal_transformer.py:39-43 SoftSplit; :94-96 FusionFeedForward), optional exact GELU fused
//   t2t_fold   : tokens [BT][L][C*k*k] -> img [BT][C][H][W]   == F.fold(x.permute(0,2,1), ...) (+ optional
//                division by fold(ones), + optional bias map)  (tfocal_transformer.py:65-72 SoftComp; :89-96 FFN)
// Both work directly on the token-major layout the Linears produce/consume, so the two 361 MB transposes, the
// normaliser divide and the GELU pass of the reference formulation disappear.  Pure HBM/L2-bound gathers:
// algorithmic bytes = tokens (BT*L*C*k*k*4) + image (BT*C*H*W*4) per call.
#include <cuda_bf16.h>
#include "common.cuh"
#include "launch.h"

namespace e2f {

__device__ __forceinline__ float gelu_exact(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f)); }
// dz * GELU'(u), GELU'(u) = Phi(u) + u phi(u): the prologue of the fold/normalise/unfold adjoint
__device__ __forceinline__ float gelu_grad(float dz, float u) {
  return dz * (0.5f * (1.0f + erff(u * 0.70710678118654752f)) + u * 0.39894228040143268f * __expf(-0.5f * u * u));
}
__device__ __forceinline__ float4 gelu_grad4(float4 dz, float4 u) {
  return make_float4(gelu_grad(dz.x, u.x), gelu_grad(dz.y, u.y), gelu_grad(dz.z, u.z), gelu_grad(dz.w, u.w));
}

// one thread per 4 consecutive token channels (float4 store); channel = c*k*k + ky*k + kx
// KC/SC/PC: compile-time kernel / stride / padding (the div/mod by 49 and 7 become multiply-shifts); KC = 0 selects
// the run-time geometry.
template <bool GELU, int KC, int SC, int PC>
__global__ void __launch_bounds__(256) t2t_unfold_kernel(const float* __restrict__ img, float* __restrict__ tok,
                                                         __nv_bfloat16* __restrict__ tok_hi,
                                                         __nv_bfloat16* __restrict__ tok_lo, int BT, int C, int H,
                                                         int W, int Kr, int Sr, int Pr, int FH, int FW) {
  const int K = KC ? KC : Kr, S = KC ? SC : Sr, P = KC ? PC : Pr;
  const int CK = C * K * K;                    // multiple of 4 is required by the launcher
  const long long total4 = static_cast<long long>(BT) * FH * FW * (CK / 4);
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i4 >= total4) return;
  const int ch0 = static_cast<int>(i4 % (CK / 4)) * 4;
  const long long t = i4 / (CK / 4);
  const int tx = static_cast<int>(t % FW);
  const int ty = static_cast<int>((t / FW) % FH);
  const long long bt = t / (static_cast<long long>(FW) * FH);
  const float* plane0 = img + bt * C * H * W;
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int ch = ch0 + e;
    const int c = ch / (K * K), kk = ch - c * K * K;
    const int ky = kk / K, kx = kk - ky * K;
    const int y = ty * S - P + ky, x = tx * S - P + kx;
    float val = 0.f;
    if (y >= 0 && y < H && x >= 0 && x < W) val = __ldg(plane0 + (static_cast<long long>(c) * H + y) * W + x);
    v[e] = GELU ? gelu_exact(val) : val;
  }
  if (tok) *reinterpret_cast<float4*>(tok + t * CK + ch0) = make_float4(v[0], v[1], v[2], v[3]);
  if (tok_hi) {   // bf16 (hi, lo) operand pair of the following Linear, written instead of / next to the fp32 tokens
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
    const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
    const __nv_bfloat162 l0 = __floats2bfloat162_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2bfloat162_rn(v[2] - f1.x, v[3] - f1.y);
    *reinterpret_cast<uint2*>(tok_hi + t * CK + ch0) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
    *reinterpret_cast<uint2*>(tok_lo + t * CK + ch0) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
  }
}

// Shared-memory staged unfold for the 7/3/3 geometry: one block per (8-channel chunk, token row, image).  The 7 image
// rows a token row touches are loaded once (coalesced, zero-padded, GELU applied ONCE per pixel instead of once per
// unfolded copy), then the 36 x (8*49) token values are written as fully coalesced runs (fp32 and/or bf16 split).
constexpr int U2_CC = 8;
// NHWC = true reads img as [BT][H][W][C] (channels_last storage, e.g. straight from a conv epilogue) instead of NCHW.
template <bool GELU, bool NHWC>
__global__ void __launch_bounds__(256) t2t_unfold733_kernel(const float* __restrict__ img, float* __restrict__ tok,
                                                            __nv_bfloat16* __restrict__ tok_hi,
                                                            __nv_bfloat16* __restrict__ tok_lo, int C, int H, int W,
                                                            int FH, int FW) {
  extern __shared__ float simg[];                 // [U2_CC][7][W + 6]
  const int WP = W + 6;
  const int c0 = blockIdx.x * U2_CC, ty = blockIdx.y;
  const long long bt = blockIdx.z;
  if (NHWC) {
    // one warp per image row of the 7, lanes along x; each lane reads its pixel's 8 channels (32 contiguous bytes)
    for (int r = threadIdx.x >> 5; r < 7; r += 8) {
      const int y = ty * 3 - 3 + r;
      const bool row_ok = y >= 0 && y < H;
      const float* srow = img + ((bt * H + y) * static_cast<long long>(W)) * C + c0;
      for (int xx = threadIdx.x & 31; xx < WP; xx += 32) {
        const int x = xx - 3;
        float v[U2_CC] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (row_ok && x >= 0 && x < W) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(srow + static_cast<long long>(x) * C));
          const float4 b = __ldg(reinterpret_cast<const float4*>(srow + static_cast<long long>(x) * C) + 1);
          v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
          if (GELU) {
#pragma unroll
            for (int cc = 0; cc < U2_CC; ++cc) v[cc] = gelu_exact(v[cc]);
          }
        }
#pragma unroll
        for (int cc = 0; cc < U2_CC; ++cc) simg[(cc * 7 + r) * WP + xx] = v[cc];
      }
    }
  } else {
  const float* src = img + (bt * C + c0) * static_cast<long long>(H) * W;
  // one warp per (channel, image row) of the 8 x 7 rows, lanes along x: no per-element index arithmetic
  for (int rr = threadIdx.x >> 5; rr < U2_CC * 7; rr += 8) {
    const int cc = rr / 7, r = rr - cc * 7;
    const int y = ty * 3 - 3 + r;
    const bool row_ok = y >= 0 && y < H;
    const float* srow = src + (static_cast<long long>(cc) * H + y) * W;
    for (int xx = threadIdx.x & 31; xx < WP; xx += 32) {
      const int x = xx - 3;
      float v = 0.f;
      if (row_ok && x >= 0 && x < W) {
        v = __ldg(srow + x);
        if (GELU) v = gelu_exact(v);
      }
      simg[rr * WP + xx] = v;
    }
  }
  }
  // thread -> fixed float4 slot q4 of a token's 8*49-value run: the (channel, ky, kx) decode happens once per thread;
  // 98 slots x 2 tokens in flight per pass (196 of 256 threads active)
  constexpr int RUN4 = U2_CC * 49 / 4, TSUB = 256 / RUN4;
  const int q4 = threadIdx.x % RUN4, tsub = threadIdx.x / RUN4;
  int off[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int q = q4 * 4 + e;
    const int cc = q / 49, kk = q - cc * 49;
    const int ky = kk / 7;
    off[e] = (cc * 7 + ky) * WP + (kk - ky * 7);
  }
  __syncthreads();
  const int CK = C * 49;
  const long long tok0 = (bt * FH + ty) * static_cast<long long>(FW);
  for (int tx = tsub; tx < (tsub < TSUB ? FW : 0); tx += TSUB) {
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = simg[tx * 3 + off[e]];
    const long long dst = (tok0 + tx) * CK + c0 * 49 + q4 * 4;
    if (tok) *reinterpret_cast<float4*>(tok + dst) = make_float4(v[0], v[1], v[2], v[3]);
    if (tok_hi) {
      const __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
      const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
      const __nv_bfloat162 l0 = __floats2bfloat162_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2bfloat162_rn(v[2] - f1.x, v[3] - f1.y);
      *reinterpret_cast<uint2*>(tok_hi + dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
      *reinterpret_cast<uint2*>(tok_lo + dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
    }
  }
}

// Shared-memory fold for the 7/3/3 geometry, used two ways:
//   FUSED  = true : fold -> / fold(ones) -> unfold -> GELU of the fusion feed-forward (tfocal_transformer.py:89-96);
//                   the folded image never goes to HBM.  Block = (CC-channel chunk, band of TR token rows, image).
//   FUSED  = false: fold (-> / fold(ones)) (+ bias map) of SoftComp (tfocal_transformer.py:65-72) and of the generic
//                   e2f_t2t_fold.  Block = (CC-channel chunk, band of 3*TR image rows, image).
// Steps:
//   1. the CC*49 values of every token whose patch touches the band are read ONCE, fully coalesced (float4), and
//      added into the band's folded image in shared memory.  Tokens are visited in 9 phases (ty mod 3, tx mod 3):
//      patches of one phase are disjoint (stride 3 * 3 >= 7), so plain += suffices — no atomics, deterministic;
//   2. every pixel is divided by its patch count (and passed through GELU / gets its bias) once;
//   3. FUSED: the TR x FW tokens of the band are written as coalesced runs (bf16 hi/lo operand pair and/or fp32).
// Algorithmic bytes: tokens in (x (TR+4)/TR or (TR+2)/TR halo re-read, served by L2) + tokens / image out.
// OUT_NHWC (fold only): the image is written channels_last, [BT][H][W][C], with an optional residual of the same
// layout added (enc_feat + trans_feat of e2fgvi.py:263 folded into the store) — the layout the decoder's convs read.
// Training (FUSED only): `u_out` non-null also writes the normalised values before GELU, [BT][L][C*49] fp32 (GELU is then
// applied at the store); BWD reads `gu` (that u, same layout as tin) and folds tin * GELU'(gu) instead of tin: the
// operator unfold . (/ fold(ones)) . fold is self-adjoint, so this is the input gradient of the training forward.
template <bool FUSED, bool GELU, int CC, bool OUT_NHWC = false, bool BWD = false>
__global__ void __launch_bounds__(256, 3) t2t_fold733_kernel(const float* __restrict__ tin, float* __restrict__ tok,
                                                          __nv_bfloat16* __restrict__ tok_hi,
                                                          __nv_bfloat16* __restrict__ tok_lo, float* __restrict__ img,
                                                          const float* __restrict__ bias, int normalize, int C, int H,
                                                          int W, int FH, int FW, int TR, int CKP,
                                                          const float* __restrict__ residual = nullptr,
                                                          const float* __restrict__ gu = nullptr,
                                                          float* __restrict__ u_out = nullptr) {
  extern __shared__ float simg[];                  // [CC][ROWS][WP], x padded by 3 on both sides; then nx[WP]
  constexpr int RUN4 = CC * 49 / 4;
  const int WP = W + 6, ROWS = FUSED ? 3 * TR + 4 : 3 * TR;
  int* nxtab = reinterpret_cast<int*>(simg + CC * ROWS * WP);
  float* rnx = reinterpret_cast<float*>(nxtab + WP);                 // 1 / nxtab (0 outside the image)
  const int c0 = blockIdx.x * CC, band = blockIdx.y;
  const long long bt = blockIdx.z;
  const int ty0 = band * TR;                       // FUSED: first token row of the band
  const int tr = min(TR, FH - ty0);
  const int ybase = FUSED ? 3 * ty0 - 3 : 3 * TR * band;   // image row held by smem row 0
  const int CK = C * 49;
  {
    float4* z = reinterpret_cast<float4*>(simg);   // CC * ROWS * WP * 4 bytes is a multiple of 16 (CC % 4 == 0)
    for (int i = threadIdx.x; i < CC * ROWS * WP / 4; i += blockDim.x) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int xx = threadIdx.x; xx < WP; xx += blockDim.x) {
      const int x = xx - 3;                        // #token columns covering x: tx in [ceil((x-3)/3), floor((x+3)/3)]
      const int nx = (x >= 0 && x < W) ? min(FW - 1, (x + 3) / 3) - max(0, (x - 1) / 3) + 1 : 0;
      nxtab[xx] = nx;
      rnx[xx] = nx ? 1.0f / static_cast<float>(nx) : 0.f;
    }
  }
  // thread -> fixed float4 slot q4 of a token's CC*49 run, so the (channel, ky, kx) decode happens once per thread:
  // RUN4 = 49 slots x TSUB tokens in flight per pass (245 of 256 threads active)
  constexpr int TSUB = 256 / RUN4;
  const int q4 = threadIdx.x % RUN4, tsub = threadIdx.x / RUN4;
  const bool active = tsub < TSUB;
  int off[4], kyv[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int q = q4 * 4 + e;
    const int cc = q / 49, kk = q - cc * 49;
    kyv[e] = kk / 7;
    off[e] = (cc * ROWS + kyv[e]) * WP + (kk - kyv[e] * 7);
  }
  __syncthreads();
  // token rows whose patches touch image rows [ybase, ybase + ROWS)
  const int tin_lo = FUSED ? max(0, ty0 - 2) : max(0, TR * band - 1);
  const int tin_hi = FUSED ? min(FH - 1, ty0 + tr + 1) : min(FH - 1, TR * band + TR);
  const float* src = tin + bt * FH * FW * static_cast<long long>(CK) + c0 * 49;
  // Row-structured walk (round 2).  ncu of the first version: 64-95 thread instructions per folded float4, almost all of
  // them per-token index / 64-bit address / predicate arithmetic.  Here a thread owns the tokens tsub, tsub + TSUB,
  // tsub + 2 TSUB (U = 3 slots; more segments only for images wider than 45 tokens) of every token row of the phase and
  // walks DOWN the rows: the global pointer and the four shared-memory pointers (one per element of its float4) advance
  // by constants, slot offsets are immediates, slot liveness is per phase and the "patches entirely inside the band"
  // test per row.  A row's read-modify-writes are issued as loads-then-stores (patches of a phase are disjoint), and
  // the NEXT row's global loads are in flight while the current row is folded (register double buffer).
  constexpr int U = 3;
  const long long gslot = 3ll * TSUB * CK, grow = 3ll * FW * CK;     // floats between slots / phase rows
  const int srow = 9 * WP;                                           // floats between phase rows in the band image
  for (int phase = 0; phase < 9; ++phase) {
    const int a = phase / 3, b = phase - 3 * a;
    const int first_ty = tin_lo + (a - tin_lo % 3 + 3) % 3;
    const int ntx = b < FW ? (FW - 1 - b) / 3 + 1 : 0;
    const int nrows = first_ty <= tin_hi ? (tin_hi - first_ty) / 3 + 1 : 0;
    for (int ts = tsub; active && ts < ntx && nrows > 0; ts += U * TSUB) {
      const bool live1 = ts + TSUB < ntx, live2 = ts + 2 * TSUB < ntx;
      const float* g = src + (static_cast<long long>(first_ty) * FW + b + 3 * ts) * CK + q4 * 4;
      int r0 = 3 * first_ty - 3 - ybase;                    // smem row of the patches' first row (may lie outside the band)
      float* se[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) se[e] = simg + (r0 * WP + 3 * b + 9 * ts + off[e]);
      auto load = [&](float4 (&v)[U], const float* gp) {
        v[0] = __ldg(reinterpret_cast<const float4*>(gp));
        if (live1) v[1] = __ldg(reinterpret_cast<const float4*>(gp + gslot));
        if (live2) v[2] = __ldg(reinterpret_cast<const float4*>(gp + 2 * gslot));
        if constexpr (BWD) {
          const float* up = gu + (gp - tin);
          v[0] = gelu_grad4(v[0], __ldg(reinterpret_cast<const float4*>(up)));
          if (live1) v[1] = gelu_grad4(v[1], __ldg(reinterpret_cast<const float4*>(up + gslot)));
          if (live2) v[2] = gelu_grad4(v[2], __ldg(reinterpret_cast<const float4*>(up + 2 * gslot)));
        }
      };
      auto foldrow = [&](const float4 (&v)[U]) {
        if (r0 >= 0 && r0 + 7 <= ROWS) {                    // no per-element row checks
          float c0v[4], c1v[4], c2v[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) c0v[e] = se[e][0];
          if (live1) {
#pragma unroll
            for (int e = 0; e < 4; ++e) c1v[e] = se[e][9 * TSUB];
          }
          if (live2) {
#pragma unroll
            for (int e = 0; e < 4; ++e) c2v[e] = se[e][18 * TSUB];
          }
          se[0][0] = c0v[0] + v[0].x; se[1][0] = c0v[1] + v[0].y; se[2][0] = c0v[2] + v[0].z; se[3][0] = c0v[3] + v[0].w;
          if (live1) {
            se[0][9 * TSUB] = c1v[0] + v[1].x; se[1][9 * TSUB] = c1v[1] + v[1].y;
            se[2][9 * TSUB] = c1v[2] + v[1].z; se[3][9 * TSUB] = c1v[3] + v[1].w;
          }
          if (live2) {
            se[0][18 * TSUB] = c2v[0] + v[2].x; se[1][18 * TSUB] = c2v[1] + v[2].y;
            se[2][18 * TSUB] = c2v[2] + v[2].z; se[3][18 * TSUB] = c2v[3] + v[2].w;
          }
        } else {
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (u == 0 || (u == 1 ? live1 : live2)) {
              const float w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int r = r0 + kyv[e];
                if (r >= 0 && r < ROWS) se[e][9 * TSUB * u] += w[e];
              }
            }
          }
        }
      };
      auto next_row = [&]() {
        g += grow;
        r0 += 9;
#pragma unroll
        for (int e = 0; e < 4; ++e) se[e] += srow;
      };
      float4 va[U], vb[U];
      load(va, g);
      for (int i = 0;;) {
        const bool more1 = i + 1 < nrows;
        if (more1) load(vb, g + grow);
        foldrow(va);
        if (!more1) break;
        next_row();
        const bool more2 = i + 2 < nrows;
        if (more2) load(va, g + grow);
        foldrow(vb);
        if (!more2) break;
        next_row();
        i += 2;
      }
    }
    __syncthreads();
  }
  // per pixel: / patch count = (#token rows covering y) * (#token columns covering x); then GELU (FUSED) or the store
  // of the image row (+ bias).  One warp per (channel, row), lanes along x.
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (!FUSED && OUT_NHWC) {
    // channels_last store: one warp per image row, each lane writes its pixel's CC channels (CC * 4 contiguous bytes)
    for (int r = warp; r < ROWS; r += 8) {
      const int y = ybase + r;
      if (y >= H) break;
      const int ny = min(FH - 1, (y + 3) / 3) - max(0, (y - 1) / 3) + 1;
      for (int x = lane; x < W; x += 32) {
        const long long pix = (bt * H + y) * static_cast<long long>(W) + x;
        float v[CC];
#pragma unroll
        for (int cc = 0; cc < CC; ++cc) {
          float t = simg[(cc * ROWS + r) * WP + x + 3];
          if (normalize) t = t / static_cast<float>(ny * nxtab[x + 3]);
          if (bias) t += __ldg(bias + (static_cast<long long>(c0 + cc) * H + y) * W + x);
          v[cc] = t;
        }
        if (residual) {
#pragma unroll
          for (int j = 0; j < CC / 4; ++j) {
            const float4 rr = __ldg(reinterpret_cast<const float4*>(residual + pix * C + c0) + j);
            v[4 * j] += rr.x; v[4 * j + 1] += rr.y; v[4 * j + 2] += rr.z; v[4 * j + 3] += rr.w;
          }
        }
#pragma unroll
        for (int j = 0; j < CC / 4; ++j)
          reinterpret_cast<float4*>(img + pix * C + c0)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
      }
    }
    return;
  }
  for (int rr = warp, cc = 0, r = warp; rr < CC * ROWS; rr += 8, r += 8) {
    while (r >= ROWS) {
      r -= ROWS;
      ++cc;
    }
    const int y = ybase + r;
    float* row = simg + rr * WP;
    if (y < 0 || y >= H) {
      if (FUSED)
        for (int xx = lane; xx < WP; xx += 32) row[xx] = 0.f;
      continue;
    }
    const int ny = min(FH - 1, (y + 3) / 3) - max(0, (y - 1) / 3) + 1;     // ty in [ceil((y-3)/3), floor((y+3)/3)]
    if (FUSED) {
      // x (1/ny)(1/nx) instead of / (ny nx): <= 1.5 ulp from the reference's fp32 division, no IEEE-division sequence and
      // no branch (columns outside the image hold finite partial sums and get the factor 0; GELU(0) = 0)
      const float rny = 1.0f / static_cast<float>(ny);
      for (int xx = lane; xx < WP; xx += 32) {
        float v = row[xx] * (rny * rnx[xx]);
        if (GELU && !u_out) v = gelu_exact(v);
        row[xx] = v;
      }
    } else {
      const long long plane = ((bt * C + c0 + cc) * H + y) * static_cast<long long>(W);
      const float* brow = bias ? bias + (static_cast<long long>(c0 + cc) * H + y) * W : nullptr;
      for (int x = lane; x < W; x += 32) {
        float v = row[x + 3];
        if (normalize) v = v / static_cast<float>(ny * nxtab[x + 3]);
        if (brow) v += __ldg(brow + x);
        img[plane + x] = v;
      }
    }
  }
  if (!FUSED) return;
  __syncthreads();
  const long long tok0 = (bt * FH + ty0) * static_cast<long long>(FW);
  if (active) {
    // thread = (float4 slot q4, token column tsub + k TSUB); pointers advance by constants (see the fold loop)
    const long long dstep = static_cast<long long>(TSUB) * CKP;          // CKP: output row pitch (>= C*49)
    for (int iy = 0; iy < tr; ++iy) {
      const float* pe[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) pe[e] = simg + (3 * iy * WP + 3 * tsub + off[e]);
      long long dst = (tok0 + static_cast<long long>(iy) * FW + tsub) * CKP + c0 * 49 + q4 * 4;
      for (int tx = tsub; tx < FW; tx += TSUB, dst += dstep) {
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[e] = *pe[e];
          pe[e] += 3 * TSUB;
        }
        if (GELU && u_out) {
          const long long du = (tok0 + static_cast<long long>(iy) * FW + tx) * CK + c0 * 49 + q4 * 4;
          *reinterpret_cast<float4*>(u_out + du) = make_float4(v[0], v[1], v[2], v[3]);
#pragma unroll
          for (int e = 0; e < 4; ++e) v[e] = gelu_exact(v[e]);
        }
        if (tok) *reinterpret_cast<float4*>(tok + dst) = make_float4(v[0], v[1], v[2], v[3]);
        if (tok_hi) {
          const __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
          const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
          const __nv_bfloat162 l0 = __floats2bfloat162_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2bfloat162_rn(v[2] - f1.x, v[3] - f1.y);
          *reinterpret_cast<uint2*>(tok_hi + dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
          *reinterpret_cast<uint2*>(tok_lo + dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
        }
      }
    }
  }
  // padded rows: the block of the last channel chunk zeroes columns [C*49, CKP) of its tokens (a following GEMM
  // multiplies them by zero weights, so they only have to be finite — zeros keep the buffer deterministic)
  if (CKP > CK && blockIdx.x == gridDim.x - 1) {
    const int padw = (CKP - CK) / 4;                             // both are multiples of 4
    for (int i = threadIdx.x; i < tr * FW * padw; i += blockDim.x) {
      const int t = i / padw, j = i - t * padw;
      const long long dst = (tok0 + t) * CKP + CK + 4 * j;
      if (tok) *reinterpret_cast<float4*>(tok + dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tok_hi) {
        *reinterpret_cast<uint2*>(tok_hi + dst) = make_uint2(0u, 0u);
        *reinterpret_cast<uint2*>(tok_lo + dst) = make_uint2(0u, 0u);
      }
    }
  }
}

// one thread per image element (c, y, x): sums the <= ceil(K/S)^2 patch entries that cover it
template <int KC, int SC, int PC>
__global__ void __launch_bounds__(256) t2t_fold_kernel(const float* __restrict__ tok, const float* __restrict__ bias,
                                                       float* __restrict__ img, int BT, int C, int H, int W, int Kr,
                                                       int Sr, int Pr, int FH, int FW, int normalize) {
  const int K = KC ? KC : Kr, S = KC ? SC : Sr, P = KC ? PC : Pr;
  const long long total = static_cast<long long>(BT) * C * H * W;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = static_cast<int>(i % W);
  const int y = static_cast<int>((i / W) % H);
  const int c = static_cast<int>((i / (static_cast<long long>(W) * H)) % C);
  const long long bt = i / (static_cast<long long>(W) * H * C);
  const int CK = C * K * K;
  // patches (ty, ky) with ty*S - P + ky == y, 0 <= ky < K
  const int ty_hi = min(FH - 1, (y + P) / S);
  const int ty_lo = max(0, (y + P - K + S) / S);     // ceil((y + P - K + 1) / S) for non-negative numerators
  const int tx_hi = min(FW - 1, (x + P) / S);
  const int tx_lo = max(0, (x + P - K + S) / S);
  float acc = 0.f;
  int count = 0;
  const float* base = tok + bt * FH * FW * CK + c * K * K;
  for (int ty = ty_lo; ty <= ty_hi; ++ty) {
    const int ky = y + P - ty * S;
    if (ky < 0 || ky >= K) continue;
    for (int tx = tx_lo; tx <= tx_hi; ++tx) {
      const int kx = x + P - tx * S;
      if (kx < 0 || kx >= K) continue;
      acc += __ldg(base + static_cast<long long>(ty * FW + tx) * CK + ky * K + kx);
      ++count;
    }
  }
  if (normalize) acc = acc / static_cast<float>(count);   // == / fold(ones); count >= 1 whenever P <= K-S... checked on host
  if (bias) acc += __ldg(bias + (static_cast<long long>(c) * H + y) * W + x);
  img[i] = acc;
}

int launch_t2t_unfold(const float* img, float* tok, void* tok_hi_v, void* tok_lo_v, int bt, int c, int h, int w, int k,
                      int s, int p, int gelu, int nhwc, cudaStream_t stream) {
  __nv_bfloat16* tok_hi = static_cast<__nv_bfloat16*>(tok_hi_v);
  __nv_bfloat16* tok_lo = static_cast<__nv_bfloat16*>(tok_lo_v);
  const int fh = (h + 2 * p - k) / s + 1, fw = (w + 2 * p - k) / s + 1;
  const long long total4 = static_cast<long long>(bt) * fh * fw * (c * k * k / 4);
  if (total4 == 0) return 0;
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total4 + threads - 1) / threads);
  const bool fast = (k == 7 && s == 3 && p == 3);
  const int smem2 = U2_CC * 7 * (w + 6) * 4;
  if (fast && c % U2_CC == 0 && smem2 <= 200 * 1024 && fh <= 65535 && bt <= 65535) {
    static DeviceOnce cfg;
    if (const int e = configure_once(cfg, 200 * 1024, t2t_unfold733_kernel<true, false>, t2t_unfold733_kernel<false, false>,
                                     t2t_unfold733_kernel<true, true>, t2t_unfold733_kernel<false, true>))
      return e;
    const dim3 grid(c / U2_CC, fh, bt);
    if (gelu && nhwc)
      t2t_unfold733_kernel<true, true><<<grid, threads, smem2, stream>>>(img, tok, tok_hi, tok_lo, c, h, w, fh, fw);
    else if (gelu)
      t2t_unfold733_kernel<true, false><<<grid, threads, smem2, stream>>>(img, tok, tok_hi, tok_lo, c, h, w, fh, fw);
    else if (nhwc)
      t2t_unfold733_kernel<false, true><<<grid, threads, smem2, stream>>>(img, tok, tok_hi, tok_lo, c, h, w, fh, fw);
    else
      t2t_unfold733_kernel<false, false><<<grid, threads, smem2, stream>>>(img, tok, tok_hi, tok_lo, c, h, w, fh, fw);
    count_launch();
    return static_cast<int>(cudaGetLastError());
  }
  if (nhwc) return -2;                               // channels_last input: only the staged 7/3/3 kernel reads it
  if (gelu && fast)
    t2t_unfold_kernel<true, 7, 3, 3><<<blocks, threads, 0, stream>>>(img, tok, tok_hi, tok_lo, bt, c, h, w, k, s, p, fh, fw);
  else if (fast)
    t2t_unfold_kernel<false, 7, 3, 3><<<blocks, threads, 0, stream>>>(img, tok, tok_hi, tok_lo, bt, c, h, w, k, s, p, fh, fw);
  else if (gelu)
    t2t_unfold_kernel<true, 0, 0, 0><<<blocks, threads, 0, stream>>>(img, tok, tok_hi, tok_lo, bt, c, h, w, k, s, p, fh, fw);
  else
    t2t_unfold_kernel<false, 0, 0, 0><<<blocks, threads, 0, stream>>>(img, tok, tok_hi, tok_lo, bt, c, h, w, k, s, p, fh, fw);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------------------
// FFN middle, second generation (round 2): fold -> / fold(ones) -> (GELU) -> unfold of FusionFeedForward
// (tfocal_transformer.py:89-96) for the 7/3/3 geometry, one block per (4-channel chunk x token-column tile, token-row band,
// image).  The first-generation kernel executed 200 M warp instructions per launch for 90 M elements, 53 %
// of them integer / predicate arithmetic (per-token divisions, per-element band checks), issue slots 68 % busy at 24 %
// occupancy — instruction-bound, 0.37 of the HBM peak; on the HQ shapes the full-width image left one block per SM
// (0.18).  Changes:
//   * the band's image in shared memory carries 2 token rows / columns of MARGIN on every side, so every patch of every
//     token that touches the tile lands inside it: the fold is 4 x (LDS, FADD, STS) per float4 with NO bounds checks;
//   * token coordinates advance incrementally (no divisions); loads of the next batch are issued before the current
//     batch is folded (register double buffer);
//   * wide images are tiled in x (<= 36 token columns per tile), so the shared-memory footprint — and 2 blocks per SM —
//     no longer depend on the image width.
// Tokens are visited in 9 phases (ty mod 3, tx mod 3): patches of one phase are disjoint (stride 3 * 3 >= 7), so plain
// read-modify-writes suffice — no atomics, deterministic.
constexpr int MID_CC = 4, MID_RUN4 = MID_CC * 49 / 4, MID_TSUB = 256 / MID_RUN4, MID_U = 4;

// u_out / BWD / gu: the training forward and the adjoint, as in t2t_fold733_kernel.
template <bool GELU, bool BWD = false>
__global__ void __launch_bounds__(256, 2) t2t_ffn_mid_kernel(const float* __restrict__ tin, float* __restrict__ tok,
                                                             __nv_bfloat16* __restrict__ tok_hi,
                                                             __nv_bfloat16* __restrict__ tok_lo, int C, int H, int W, int FH,
                                                             int FW, int TR, int TW, int XT, int CKP,
                                                             const float* __restrict__ gu = nullptr,
                                                             float* __restrict__ u_out = nullptr) {
  extern __shared__ float simg[];                  // [CC][R][WP] + int ny[R] + int nx[WP]
  const int chunk = blockIdx.x / XT, xt = blockIdx.x - chunk * XT;
  const int c0 = chunk * MID_CC;
  const long long bt = blockIdx.z;
  const int ty0 = blockIdx.y * TR, tx0 = xt * TW;                       // first OUTPUT token of the tile
  const int tr = min(TR, FH - ty0), tw = min(TW, FW - tx0);
  const int R = 3 * (TR + 4) + 4, WP = 3 * (TW + 4) + 4;                // image rows / columns held (incl. margins)
  const int tyb = ty0 - 2, txb = tx0 - 2;                               // token whose patch starts at smem row / col 0
  int* nytab = reinterpret_cast<int*>(simg + MID_CC * R * WP);
  int* nxtab = nytab + R;
  const int CK = C * 49;
  {
    float4* z = reinterpret_cast<float4*>(simg);                        // CC * R * WP * 4 bytes is a multiple of 16
    for (int i = threadIdx.x; i < MID_CC * R * WP / 4; i += 256) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    // number of token rows / columns whose patch covers image row y / column x (0 outside the image)
    for (int r = threadIdx.x; r < R; r += 256) {
      const int y = 3 * tyb - 3 + r;
      nytab[r] = (y >= 0 && y < H) ? max(0, min(FH - 1, (y + 3) / 3) - max(0, (y - 1) / 3) + 1) : 0;
    }
    for (int cc = threadIdx.x; cc < WP; cc += 256) {
      const int x = 3 * txb - 3 + cc;
      nxtab[cc] = (x >= 0 && x < W) ? max(0, min(FW - 1, (x + 3) / 3) - max(0, (x - 1) / 3) + 1) : 0;
    }
  }
  // thread -> fixed float4 slot q4 of a token's CC*49 run (49 slots) x token lane tsub (5 lanes; 245 of 256 threads)
  const int q4 = threadIdx.x % MID_RUN4, tsub = threadIdx.x / MID_RUN4;
  const bool active = tsub < MID_TSUB;
  int off[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int q = q4 * 4 + e;
    const int cc = q / 49, kk = q - cc * 49;
    const int ky = kk / 7;
    off[e] = (cc * R + ky) * WP + (kk - ky * 7);
  }
  __syncthreads();
  // input tokens whose patches touch the tile's output patches
  const int ty_lo = max(0, tyb), ty_hi = min(FH - 1, ty0 + tr + 1);
  const int tx_lo = max(0, txb), tx_hi = min(FW - 1, tx0 + tw + 1);
  const float* src = tin + bt * FH * FW * static_cast<long long>(CK) + c0 * 49 + q4 * 4;
  for (int phase = 0; phase < 9; ++phase) {
    const int a = phase / 3, b = phase - 3 * a;
    const int fy = ty_lo + (a - ty_lo % 3 + 3) % 3, fx = tx_lo + (b - tx_lo % 3 + 3) % 3;   // first token of the phase
    const int nty = fy <= ty_hi ? (ty_hi - fy) / 3 + 1 : 0, ntx = fx <= tx_hi ? (tx_hi - fx) / 3 + 1 : 0;
    const int ntok = active ? nty * ntx : 0;
    // this thread's tokens: linear index t = tsub, tsub + TSUB, ... over the (nty x ntx) grid, advanced incrementally
    int iy = 0, ix = tsub;
    while (ntx > 0 && ix >= ntx) { ix -= ntx; ++iy; }
    auto advance = [&]() {
      ix += MID_TSUB;
      while (ix >= ntx) { ix -= ntx; ++iy; }
    };
    float4 va[MID_U], vb[MID_U];
    int ba[MID_U], bb[MID_U];
    auto issue = [&](int t, float4 (&v4)[MID_U], int (&base)[MID_U]) {
#pragma unroll
      for (int u = 0; u < MID_U; ++u) {
        if (t + u * MID_TSUB < ntok) {
          const int ty = fy + 3 * iy, tx = fx + 3 * ix;
          v4[u] = __ldg(reinterpret_cast<const float4*>(src + static_cast<long long>(ty * FW + tx) * CK));
          if constexpr (BWD)
            v4[u] = gelu_grad4(v4[u], __ldg(reinterpret_cast<const float4*>(gu + (src - tin) +
                                                                              static_cast<long long>(ty * FW + tx) * CK)));
          base[u] = 3 * (ty - tyb) * WP + 3 * (tx - txb);
          advance();
        }
      }
    };
    auto fold = [&](int t, const float4 (&v4)[MID_U], const int (&base)[MID_U]) {
      float cur[MID_U][4];
#pragma unroll
      for (int u = 0; u < MID_U; ++u) {
        if (t + u * MID_TSUB < ntok) {
#pragma unroll
          for (int e = 0; e < 4; ++e) cur[u][e] = simg[base[u] + off[e]];
        }
      }
#pragma unroll
      for (int u = 0; u < MID_U; ++u) {
        if (t + u * MID_TSUB < ntok) {
          simg[base[u] + off[0]] = cur[u][0] + v4[u].x;
          simg[base[u] + off[1]] = cur[u][1] + v4[u].y;
          simg[base[u] + off[2]] = cur[u][2] + v4[u].z;
          simg[base[u] + off[3]] = cur[u][3] + v4[u].w;
        }
      }
    };
    int t = tsub;
    if (t < ntok) issue(t, va, ba);
    while (t < ntok) {
      const int n1 = t + MID_TSUB * MID_U;
      if (n1 < ntok) issue(n1, vb, bb);
      fold(t, va, ba);
      t = n1;
      if (t >= ntok) break;
      const int n2 = t + MID_TSUB * MID_U;
      if (n2 < ntok) issue(n2, va, ba);
      fold(t, vb, bb);
      t = n2;
    }
    __syncthreads();
  }
  // per pixel: / (#token rows covering y) * (#token columns covering x), GELU; pixels outside the image (and pixels
  // no patch covers) become exact zeros — they are the unfold's zero padding.  One warp per (channel, row).
  // Only rows / columns [6, 3*t + 13) are read by the tile's output patches (the margins only absorb stray patch rows).
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nr = 3 * tr + 7, ncol = 3 * tw + 7;
  for (int rr = warp; rr < MID_CC * nr; rr += 8) {
    const int cc = rr / nr, r = rr - cc * nr + 6;
    float* row = simg + (cc * R + r) * WP;
    const int ny = nytab[r];
    for (int xx = 6 + lane; xx < 6 + ncol; xx += 32) {
      const int cnt = ny * nxtab[xx];
      float v = 0.f;
      if (cnt) {
        v = row[xx] / static_cast<float>(cnt);
        if (GELU && !u_out) v = gelu_exact(v);
      }
      row[xx] = v;
    }
  }
  __syncthreads();
  // unfold: the tr x tw tokens of the tile as coalesced runs (bf16 hi/lo operand pair and/or fp32)
  {
    const int nout = active ? tr * tw : 0;
    int iy = 0, ix = tsub;
    while (tw > 0 && ix >= tw) { ix -= tw; ++iy; }
    for (int t = tsub; t < nout; t += MID_TSUB) {
      const int base = 3 * (iy + 2) * WP + 3 * (ix + 2);
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = simg[base + off[e]];
      const long long dst = ((bt * FH + ty0 + iy) * static_cast<long long>(FW) + tx0 + ix) * CKP + c0 * 49 + q4 * 4;
      if (GELU && u_out) {
        const long long du = ((bt * FH + ty0 + iy) * static_cast<long long>(FW) + tx0 + ix) * CK + c0 * 49 + q4 * 4;
        *reinterpret_cast<float4*>(u_out + du) = make_float4(v[0], v[1], v[2], v[3]);
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = gelu_exact(v[e]);
      }
      if (tok) *reinterpret_cast<float4*>(tok + dst) = make_float4(v[0], v[1], v[2], v[3]);
      if (tok_hi) {
        const __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
        const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
        const __nv_bfloat162 l0 = __floats2bfloat162_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2bfloat162_rn(v[2] - f1.x, v[3] - f1.y);
        *reinterpret_cast<uint2*>(tok_hi + dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
        *reinterpret_cast<uint2*>(tok_lo + dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
      }
      ix += MID_TSUB;
      while (ix >= tw) { ix -= tw; ++iy; }
    }
  }
  // padded rows: the block of the last channel chunk zeroes columns [C*49, CKP) of its tokens (a following GEMM
  // multiplies them by zero weights, so they only have to be finite — zeros keep the buffer deterministic)
  if (CKP > CK && chunk == C / MID_CC - 1) {
    const int padw = (CKP - CK) / 4;                             // both are multiples of 4
    for (int i = threadIdx.x; i < tr * tw * padw; i += 256) {
      const int tk = i / padw, j = i - tk * padw;
      const int iy = tk / tw, ix = tk - iy * tw;
      const long long dst = ((bt * FH + ty0 + iy) * static_cast<long long>(FW) + tx0 + ix) * CKP + CK + 4 * j;
      if (tok) *reinterpret_cast<float4*>(tok + dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tok_hi) {
        *reinterpret_cast<uint2*>(tok_hi + dst) = make_uint2(0u, 0u);
        *reinterpret_cast<uint2*>(tok_lo + dst) = make_uint2(0u, 0u);
      }
    }
  }
}

// Band height (in token rows) of t2t_fold733_kernel and its dynamic shared memory: the tallest band that keeps 3 blocks
// per SM; wide images (few rows fit) take up to 200 KB instead.  rows(tr) = 3*tr + extra image rows.  0 = does not fit.
static int fold733_band(int w, int fh, int extra_rows, size_t* smem, int CC = 4, long long blocks_per_band = 0) {
  const size_t row_bytes = static_cast<size_t>(CC) * (w + 6) * sizeof(float), tab = 2 * (w + 6) * sizeof(int);   // nxtab + rnx
  auto band_rows = [&](size_t budget) {
    const long long rows = static_cast<long long>((budget - tab) / row_bytes) - extra_rows;
    return rows < 3 ? 0 : static_cast<int>(rows / 3);
  };
  int tr = band_rows(72 * 1024);
  if (tr < 5 && tr < fh) tr = band_rows(200 * 1024);
  if (tr < 1) return 0;
  tr = tr < fh ? tr : fh;
  int bands = (fh + tr - 1) / tr;
  // few images (one clip per call): a band is walked serially by one block, so shorter bands until every SM holds two
  // blocks (the extra halo re-reads are L2 hits): 66 -> ~40 us per launch at one clip
  while (blocks_per_band > 0 && bands * blocks_per_band < 2ll * num_sms() && (fh + bands - 1) / bands > 4) ++bands;
  tr = (fh + bands - 1) / bands;                   // even out the bands
  *smem = row_bytes * (3 * tr + extra_rows) + tab;
  return tr;
}

static int fold733_configure() {
  static DeviceOnce folds, fullwidth;
  if (const int e = configure_once(folds, 200 * 1024, t2t_fold733_kernel<false, false, 4>,
                                   t2t_fold733_kernel<false, false, 8, true>))
    return e;
  // three ~63 KB bands per SM need the large shared-memory carve-out (ncu: the default left room for two)
  return configure_once_carveout(fullwidth, 200 * 1024, cudaSharedmemCarveoutMaxShared, t2t_fold733_kernel<true, true, 4>,
                                 t2t_fold733_kernel<true, false, 4>, t2t_fold733_kernel<true, false, 4, false, true>);
}

// Fused fold/normalise/unfold(/GELU).  Returns -2 (unsupported) when the geometry is not 7/3/3 or no band fits in
// shared memory; the caller then composes launch_t2t_fold + launch_t2t_unfold.
// First-generation launch (whole image width per block): measured faster than the x-tiled kernel while the image is
// narrow enough for >= 2 blocks per SM.
static int launch_fold733_fullwidth(const float* tin, float* tok, void* tok_hi, void* tok_lo, int bt, int c, int h, int w,
                                    int fh, int fw, int gelu, int out_pitch, const float* gu, float* u_out,
                                    cudaStream_t stream) {
  constexpr int CC = 4;
  size_t smem = 0;
  const int tr = fold733_band(w, fh, 4, &smem, CC, static_cast<long long>(c / CC) * bt);
  if (tr < 1) return -2;
  auto* hi = static_cast<__nv_bfloat16*>(tok_hi);
  auto* lo = static_cast<__nv_bfloat16*>(tok_lo);
  const dim3 grid(c / CC, (fh + tr - 1) / tr, bt);
  if (const int e = fold733_configure()) return e;
  if (gu)
    t2t_fold733_kernel<true, false, CC, false, true><<<grid, 256, smem, stream>>>(tin, tok, hi, lo, nullptr, nullptr, 1, c, h, w,
                                                                                  fh, fw, tr, out_pitch, nullptr, gu);
  else if (gelu)
    t2t_fold733_kernel<true, true, CC><<<grid, 256, smem, stream>>>(tin, tok, hi, lo, nullptr, nullptr, 1, c, h, w, fh, fw, tr,
                                                                    out_pitch, nullptr, nullptr, u_out);
  else
    t2t_fold733_kernel<true, false, CC><<<grid, 256, smem, stream>>>(tin, tok, hi, lo, nullptr, nullptr, 1, c, h, w, fh, fw, tr,
                                                                     out_pitch);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_t2t_fold_unfold(const float* tin, float* tok, void* tok_hi, void* tok_lo, int bt, int c, int h, int w, int k,
                           int s, int p, int gelu, int out_pitch, cudaStream_t stream, const float* gu, float* u_out) {
  if (k != 7 || s != 3 || p != 3 || c % MID_CC) return -2;
  const int fh = (h + 2 * p - k) / s + 1, fw = (w + 2 * p - k) / s + 1;
  if (bt == 0 || fh <= 0 || fw <= 0) return 0;
  if (bt > 65535) return -2;
  if (fw <= 40)
    return launch_fold733_fullwidth(tin, tok, tok_hi, tok_lo, bt, c, h, w, fh, fw, gelu, out_pitch, gu, u_out, stream);
  // tile: <= 36 token columns (x tiles evened out) and the tallest band of token rows that keeps two blocks per SM
  const int xt = (fw + 35) / 36, tw = (fw + xt - 1) / xt;
  const int wp = 3 * (tw + 4) + 4;
  auto smem_of = [&](int tr) { return static_cast<size_t>(MID_CC) * (3 * (tr + 4) + 4) * wp * 4 + (3 * (tr + 4) + 4 + wp) * 4; };
  int tr = fh < 12 ? fh : 12;
  while (tr > 1 && smem_of(tr) > 100 * 1024) --tr;
  const int bands = (fh + tr - 1) / tr;
  tr = (fh + bands - 1) / bands;                   // even out the bands
  const size_t smem = smem_of(tr);
  if (smem > 200 * 1024 || bands > 65535) return -2;
  static DeviceOnce cfg;
  if (const int e = configure_once(cfg, 200 * 1024, t2t_ffn_mid_kernel<true>, t2t_ffn_mid_kernel<false>,
                                   t2t_ffn_mid_kernel<false, true>))
    return e;
  auto* hi = static_cast<__nv_bfloat16*>(tok_hi);
  auto* lo = static_cast<__nv_bfloat16*>(tok_lo);
  const dim3 grid((c / MID_CC) * xt, bands, bt);
  if (gu)
    t2t_ffn_mid_kernel<false, true><<<grid, 256, smem, stream>>>(tin, tok, hi, lo, c, h, w, fh, fw, tr, tw, xt, out_pitch, gu);
  else if (gelu)
    t2t_ffn_mid_kernel<true><<<grid, 256, smem, stream>>>(tin, tok, hi, lo, c, h, w, fh, fw, tr, tw, xt, out_pitch, nullptr,
                                                          u_out);
  else
    t2t_ffn_mid_kernel<false><<<grid, 256, smem, stream>>>(tin, tok, hi, lo, c, h, w, fh, fw, tr, tw, xt, out_pitch);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// fold (+ / fold(ones)) (+ bias map) (+ channels_last residual) -> channels_last image.  7/3/3 with C % 8 == 0 only (-2).
int launch_t2t_fold_nhwc(const float* tok, const float* bias, const float* residual, float* img, int bt, int c, int h,
                         int w, int k, int s, int p, int normalize, cudaStream_t stream) {
  if (k != 7 || s != 3 || p != 3 || c % 8 || bt > 65535) return -2;
  const int fh = (h + 2 * p - k) / s + 1, fw = (w + 2 * p - k) / s + 1;
  if (bt == 0) return 0;
  size_t smem = 0;
  const int tr = fold733_band(w, (h + 2) / 3, 0, &smem, 8);
  if (tr < 1) return -2;
  if (const int e = fold733_configure()) return e;
  const dim3 grid(c / 8, (h + 3 * tr - 1) / (3 * tr), bt);
  t2t_fold733_kernel<false, false, 8, true><<<grid, 256, smem, stream>>>(tok, nullptr, nullptr, nullptr, img, bias, normalize, c,
                                                                         h, w, fh, fw, tr, c * 49, residual);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int launch_t2t_fold(const float* tok, const float* bias, float* img, int bt, int c, int h, int w, int k, int s,
                    int p, int normalize, cudaStream_t stream) {
  const int fh = (h + 2 * p - k) / s + 1, fw = (w + 2 * p - k) / s + 1;
  const long long total = static_cast<long long>(bt) * c * h * w;
  if (total == 0) return 0;
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
  if (k == 7 && s == 3 && p == 3 && c % 4 == 0 && bt <= 65535) {
    // shared-memory fold: coalesced token reads, one block per (4 channels, band of 3*tr image rows, image)
    size_t smem = 0;
    const int tr = fold733_band(w, (h + 2) / 3, 0, &smem);
    if (tr >= 1) {
      if (const int e = fold733_configure()) return e;
      const dim3 grid(c / 4, (h + 3 * tr - 1) / (3 * tr), bt);
      t2t_fold733_kernel<false, false, 4><<<grid, 256, smem, stream>>>(tok, nullptr, nullptr, nullptr, img, bias, normalize, c, h,
                                                                       w, fh, fw, tr, c * 49);
      count_launch();
      return static_cast<int>(cudaGetLastError());
    }
  }
  if (k == 7 && s == 3 && p == 3)
    t2t_fold_kernel<7, 3, 3><<<blocks, threads, 0, stream>>>(tok, bias, img, bt, c, h, w, k, s, p, fh, fw, normalize);
  else
    t2t_fold_kernel<0, 0, 0><<<blocks, threads, 0, stream>>>(tok, bias, img, bt, c, h, w, k, s, p, fh, fw, normalize);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
