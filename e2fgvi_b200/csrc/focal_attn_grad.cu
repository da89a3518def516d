// Backward of the temporal focal window attention core (focal_attn.cu): given the fp16 qkv / qkv_pooled the forward
// read and dO = dL/d(attention output) in fp32, the exact-softmax gradients dq, dk, dv of the token rows and dk, dv of
// the pooled rows — the gradient of float64 autograd through the reference's literal key list.
//
// The key set of every (window, frame) is the forward's: the expanded window wrapped like torch.roll with log2(m) added
// to the logit of a position the reference lists m times, the in-grid pooled neighbours, and the zero-padded pooled
// neighbours folded into the initial (max, sum) = (-100, n_masked) (k = v = 0: they get no gradient but stay in the
// denominator).  A merged key's P already carries its multiplicity, so its dS is the sum over its copies.
//
// Three deterministic kernels, no atomics.  Every product runs on wgmma with the bf16 three-term split (hi.hi + hi.lo +
// lo.hi, fp32 accumulation): an fp16 value is exactly hi + lo, dO and the fp32 P / dS are split to 2^-17.
//   1. rows: one CTA (one warpgroup) per (64 query rows, head, window).  S = Q K^T and dP = dO V^T over the window's
//      keys give each row's log2-sum-exp and D = sum_j P_ij dP_ij by an online rescaled sum, in fp32 (not from the
//      forward's fp16 P): 2 products.
//   2. keys: one CTA (one warpgroup) per (group of key tiles, window, head).  For each of its 64-key tiles and each
//      64-query tile of the window: S^T = K Q^T, dP^T = V dO^T, P and dS in registers, written to shared memory as bf16
//      (hi, lo); dV += P^T dO and dK += dS^T Q in registers, and dS . K added to the group's dQ partial: 5 products.
//      dK | dV of the tile go to a per-(window, key slot) fp32 partial; dQ to a per-(window, group) partial.
//   3. gather: one CTA per (key token, head).  Adds the partials of every (window, key slot) that lists the token, in
//      a fixed order (expanded row, then column; pooled: window row, then column): a token reaches several windows'
//      rings (up to four, more than once through the wrap on small grids) and every pooled neighbourhood that holds it.
//      A ring token is also a query of exactly one window: its dQ is the sum of that window's GROUPS partials, in order.
// Kernels 2 and 3 run over chunks of (clip, head) units so that the partials stay within PARTIAL_BUDGET floats.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "focal_geom.cuh"
#include "launch.h"

namespace e2f {
namespace attn_grad {

using attn::MAX_RING;
constexpr int HD = 128;
constexpr int TM = 64;                         // query / key rows per tile (the wgmma M of one warpgroup)
constexpr int ATOM = TM * 128;                 // [64 rows][64 bf16] 128B-swizzled sub-tile: 8 KB
constexpr int TILE = 2 * ATOM;                 // one bf16 term of 64 rows x 128 channels
constexpr int THREADS = 128;                   // one warpgroup
constexpr int GROUPS = 8;                      // key-tile groups per (window, head): CTAs of kernel 2, dQ partials
constexpr int MAX_FRAME_KEYS = 384;
constexpr int MAX_SOURCES = 128;               // (window, key slot) pairs one token can reach
constexpr long long PARTIAL_BUDGET = 32ll << 20;   // floats of dK | dV and dQ partials per chunk (128 MB)
constexpr float LOG2E = 1.4426950408889634f;

struct Geo {
  const __half* qkv;
  const __half* pooled;
  const float* dout;
  float* dqkv;
  float* dpooled;
  float* stats;                  // [B * nW][heads][nq][2]: log2-sum-exp, D
  float* part;                   // [units in chunk][nW][NKS][2 * HD]: dK | dV partials
  float* part_dq;                // [units in chunk][nW][GROUPS][nq][HD]: dQ partials
  int B, T, H, W, heads, C;
  int wh, ww, eh, ew, fh, fw, nWh, nWw, use_pooled;
  float scale, scale_log2;
  int n1, n2, NKS;               // NKS: key-slot stride of the partials (T * (n1 + n2 + fh * fw))
  int unit0;                     // first (clip, head) unit of this chunk
  uint8_t ring_pos[MAX_RING], ring_mult[MAX_RING];
  uint8_t ring_slot[MAX_RING];   // expanded position -> its index in ring_pos (255: not listed)
};

// one window's key list: [T x n1 single ring | T x npool pooled | T x n2 multiple ring], frame-major in each part
struct Win {
  int b, wi, wj, pi0, pj0, PW, npool, n_masked, nA, nB, NK;
};

__host__ __device__ inline Win make_win(const Geo& g, int b, int win) {
  Win w;
  w.b = b;
  w.wi = win / g.nWw;
  w.wj = win % g.nWw;
  int PH = 0;
  w.pi0 = w.pj0 = w.PW = 0;
  if (g.use_pooled) {
    w.pi0 = w.wi - g.fh / 2 > 0 ? w.wi - g.fh / 2 : 0;
    w.pj0 = w.wj - g.fw / 2 > 0 ? w.wj - g.fw / 2 : 0;
    PH = (w.wi + g.fh / 2 < g.nWh - 1 ? w.wi + g.fh / 2 : g.nWh - 1) - w.pi0 + 1;
    w.PW = (w.wj + g.fw / 2 < g.nWw - 1 ? w.wj + g.fw / 2 : g.nWw - 1) - w.pj0 + 1;
  }
  w.npool = PH * w.PW;
  w.n_masked = g.use_pooled ? g.T * (g.fh * g.fw - w.npool) : 0;
  w.nA = g.T * g.n1;
  w.nB = w.nA + g.T * w.npool;
  w.NK = w.nB + g.T * g.n2;
  return w;
}

// Every (window, key slot, multiplicity) that lists key token (t, y, x) of the token grid (pooled = 0) or of the pooled
// grid (pooled = 1, (y, x) = (pi, pj)), in the gather's fixed order.  Returns the count (at most `cap`).
__host__ __device__ inline int key_sources(const Geo& g, int t, int pooled, int y, int x, int* win, int* slot, int* mult,
                                           int cap) {
  int n = 0;
  if (pooled) {
    for (int wi = y - g.fh / 2; wi <= y + g.fh / 2; ++wi)
      for (int wj = x - g.fw / 2; wj <= x + g.fw / 2; ++wj) {
        if (wi < 0 || wi >= g.nWh || wj < 0 || wj >= g.nWw || n >= cap) continue;
        const Win w = make_win(g, 0, wi * g.nWw + wj);
        win[n] = wi * g.nWw + wj;
        slot[n] = w.nA + t * w.npool + (y - w.pi0) * w.PW + (x - w.pj0);
        mult[n] = 1;
        ++n;
      }
    return n;
  }
  const int EH = g.wh + 2 * g.eh, EW = g.ww + 2 * g.ew;
  for (int er = 0; er < EH; ++er) {
    // window row wi sees token row y at expanded row er when (wi * wh - eh + er) == y modulo H
    const int rr = ((y + g.eh - er) % g.H + g.H) % g.H;
    if (rr % g.wh) continue;
    for (int ec = 0; ec < EW; ++ec) {
      const int cc = ((x + g.ew - ec) % g.W + g.W) % g.W;
      if (cc % g.ww) continue;
      const int s = g.ring_slot[er * EW + ec];
      if (s == 255 || n >= cap) continue;
      const Win w = make_win(g, 0, (rr / g.wh) * g.nWw + cc / g.ww);
      win[n] = (rr / g.wh) * g.nWw + cc / g.ww;
      slot[n] = s < g.n1 ? t * g.n1 + s : w.nB + t * g.n2 + (s - g.n1);
      mult[n] = g.ring_mult[s];
      ++n;
    }
  }
  return n;
}

struct Smem {                    // bytes; every tile 1024-aligned
  static constexpr int K = 0;                    // [hi | lo] K tile (kernel 1: dO)
  static constexpr int V = K + 2 * TILE;         // [hi | lo] V tile
  static constexpr int Q = V + 2 * TILE;         // [hi | lo] Q tile
  static constexpr int O = Q + 2 * TILE;         // [hi | lo] dO tile
  static constexpr int P = O + 2 * TILE;         // [hi | lo] P^T  [64 keys][64 queries]
  static constexpr int DS = P + 2 * ATOM;        // [hi | lo] dS^T [64 keys][64 queries]
  static constexpr int CB = DS + 2 * ATOM;       // [64] float key bias
  static constexpr int CL = CB + TM * 4;         // [64] float query log2-sum-exp
  static constexpr int CD = CL + TM * 4;         // [64] float query D
  static constexpr int FB = CD + TM * 4;         // [MAX_FRAME_KEYS] float frame-table bias
  static constexpr int FT = FB + MAX_FRAME_KEYS * 4;   // [MAX_FRAME_KEYS] int frame-table offset
  static constexpr int PTR = FT + MAX_FRAME_KEYS * 4;  // [64] uint64 row addresses
  static constexpr int BYTES = PTR + 3 * TM * 8;      // key rows | Q rows | dO rows
};
constexpr int SMEM_BYTES = Smem::BYTES + 1024;

// per-frame key table of window w: entry e -> offset (in halfs) of that key's token inside its frame, logit bias
__device__ void build_frame_table(const Geo& g, const Win& w, int* ftab, float* fbias) {
  const int EW = g.ww + 2 * g.ew;
  const int C3 = 3 * g.C;
  for (int e = threadIdx.x; e < g.n1 + w.npool + g.n2; e += THREADS) {
    int off;
    float bias = 0.f;
    if (e >= g.n1 && e < g.n1 + w.npool) {
      const int pp = e - g.n1;
      off = ((w.pi0 + pp / w.PW) * g.nWw + (w.pj0 + pp % w.PW)) * C3;
    } else {
      const int s = (e < g.n1) ? e : e - w.npool;
      const int pos = g.ring_pos[s], mult = g.ring_mult[s];
      const int er = pos / EW, ec = pos - er * EW;
      int y = (w.wi * g.wh - g.eh + er) % g.H;
      int x = (w.wj * g.ww - g.ew + ec) % g.W;
      y += (y < 0) ? g.H : 0;
      x += (x < 0) ? g.W : 0;
      off = (y * g.W + x) * C3;
      bias = (mult == 1) ? 0.f : log2f(static_cast<float>(mult));
    }
    ftab[e] = off;
    fbias[e] = bias;
  }
}

// address of key slot kk's K row (V is C halfs further) and its log2-domain logit bias; nullptr / -inf past the list
__device__ const __half* key_row(const Geo& g, const Win& w, const int* ftab, const float* fbias, int head, int kk,
                                 float& bias) {
  const size_t C3 = 3 * static_cast<size_t>(g.C);
  const size_t ring_frame = static_cast<size_t>(g.H) * g.W * C3, pool_frame = static_cast<size_t>(g.nWh) * g.nWw * C3;
  const __half* ring = g.qkv + static_cast<size_t>(w.b) * g.T * ring_frame + g.C + head * HD;
  bias = 0.f;
  if (kk < w.nA) {
    const int t = kk / g.n1, e = kk - t * g.n1;
    return ring + t * ring_frame + ftab[e];
  }
  if (kk < w.nB) {
    const int j = kk - w.nA, t = j / w.npool, e = g.n1 + (j - t * w.npool);
    return g.pooled + static_cast<size_t>(w.b) * g.T * pool_frame + g.C + head * HD + t * pool_frame + ftab[e];
  }
  if (kk < w.NK) {
    const int j = kk - w.nB, t = j / g.n2, e = g.n1 + w.npool + (j - t * g.n2);
    bias = fbias[e];
    return ring + t * ring_frame + ftab[e];
  }
  bias = -INFINITY;
  return nullptr;
}

// token index (b, t, y, x) of query qi of window w
__device__ __forceinline__ size_t query_token(const Geo& g, const Win& w, int qi) {
  const int area = g.wh * g.ww, t = qi / area, p = qi - t * area;
  const int y = w.wi * g.wh + p / g.ww, x = w.wj * g.ww + p % g.ww;
  return ((static_cast<size_t>(w.b) * g.T + t) * g.H + y) * g.W + x;
}

// 64 rows of 128 channels (address per row in ptr[], nullptr = zeros; `off` elements into each row) -> the bf16 (hi, lo)
// split as two K-major tiles [hi | lo], each two 64-channel atoms of [64 rows][128 B], 128B-swizzled.  fp16 is exact.
template <bool F32>
__device__ void fill_split(uint8_t* tile, const uint64_t* ptr, int off) {
  for (int i = threadIdx.x; i < TM * 16; i += THREADS) {
    const int row = i >> 4, ch = i & 15;
    float v[8];
    if (!ptr[row]) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = 0.f;
    } else if constexpr (F32) {
      const float* src = reinterpret_cast<const float*>(ptr[row]) + off + ch * 8;
      const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
      const uint4 raw = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(ptr[row]) + off + ch * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        v[2 * e] = f.x;
        v[2 * e + 1] = f.y;
      }
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const __nv_bfloat162 hb = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
      const float2 hf = __bfloat1622float2(hb);
      const __nv_bfloat162 lb = __floats2bfloat162_rn(v[2 * e] - hf.x, v[2 * e + 1] - hf.y);
      hi[e] = *reinterpret_cast<const uint32_t*>(&hb);
      lo[e] = *reinterpret_cast<const uint32_t*>(&lb);
    }
    const uint32_t o = (ch >> 3) * ATOM + sw128_offset(row, ch & 7);
    *reinterpret_cast<uint4*>(tile + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(tile + TILE + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

// K-major operand: k16 step k of a 128-channel tile (atom k / 4, 32 bytes per step inside it)
__device__ __forceinline__ uint64_t kdesc(uint32_t addr, int k) {
  return gmma_desc_sw128(addr, 16, 1024) + (k >> 2) * (ATOM >> 4) + 2 * (k & 3);
}
// MN-major operand [k rows][64 or 128 columns]: k16 step k = 16 rows of 128 B; the second 64-column atom ATOM further
__device__ __forceinline__ uint64_t mdesc(uint32_t addr, int k) {
  return gmma_desc_sw128(addr, ATOM, 1024) + k * (2048 >> 4);
}

// D[64 x 128] (+)= A[64 x 16] . B[16 x 128]: A K-major, B MN-major (transpose bit of B only), bf16
__device__ __forceinline__ void wgmma_n128_bf16_tb(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {" E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5
               E2F_WR6 E2F_WR7 "}, %64, %65, p, 1, 1, 0, 1;\n}\n"
               : E2F_WD64(0)
               : "l"(adesc), "l"(bdesc), "r"(acc));
}

// D[64 x 64] = A . B^T over 128 channels, both [hi | lo] K-major tiles of 64 rows: lo.hi + hi.lo + hi.hi per k16 step
__device__ __forceinline__ void mma_rows(float* d, uint32_t a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < HD / 16; ++k) {
    wgmma_ss<64, false>(d, kdesc(a + TILE, k), kdesc(b, k), k != 0);
    wgmma_ss<64, false>(d, kdesc(a, k), kdesc(b + TILE, k), 1);
    wgmma_ss<64, false>(d, kdesc(a, k), kdesc(b, k), 1);
  }
}

__device__ __forceinline__ uint8_t* aligned_smem(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
}

// ------------------------------------------------------------------------------------------------------ 1. rows
__global__ void __launch_bounds__(THREADS, 1) attn_grad_rows_kernel(const __grid_constant__ Geo g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = aligned_smem(smem_raw);
  float* kbias = reinterpret_cast<float*>(smem + Smem::CB);
  float* fbias = reinterpret_cast<float*>(smem + Smem::FB);
  int* ftab = reinterpret_cast<int*>(smem + Smem::FT);
  uint64_t* ptr = reinterpret_cast<uint64_t*>(smem + Smem::PTR);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = lane & 3;
  const int rw = 16 * warp + (lane >> 2);               // this thread's accumulator rows rw, rw + 8
  const int nW = g.nWh * g.nWw, head = blockIdx.y, bw = blockIdx.z;
  const Win w = make_win(g, bw / nW, bw % nW);
  const int nq = g.T * g.wh * g.ww, q0 = blockIdx.x * TM;
  const size_t C3 = 3 * static_cast<size_t>(g.C);
  const uint32_t sb = smem_u32(smem);

  build_frame_table(g, w, ftab, fbias);
  if (tid < TM) {
    const int qi = q0 + tid;
    const size_t tok = qi < nq ? query_token(g, w, qi) : 0;
    ptr[tid] = qi < nq ? reinterpret_cast<uint64_t>(g.qkv + tok * C3 + head * HD) : 0;
    ptr[TM + tid] = qi < nq ? reinterpret_cast<uint64_t>(g.dout + tok * g.C + head * HD) : 0;
  }
  __syncthreads();
  fill_split<false>(smem + Smem::Q, ptr, 0);
  fill_split<true>(smem + Smem::O, ptr + TM, 0);

  float m[2], l[2], a[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = w.n_masked > 0 ? -100.0f * LOG2E : -INFINITY;
    l[h] = static_cast<float>(w.n_masked);            // the padded neighbours: P = e^-100 each, dP = 0
    a[h] = 0.f;
  }
  const int num_kt = (w.NK + TM - 1) / TM;
  for (int kt = 0; kt < num_kt; ++kt) {
    __syncthreads();                                   // the previous tile's MMAs are done with K, V, ptr, kbias
    if (tid < TM) {
      float bias;
      ptr[tid] = reinterpret_cast<uint64_t>(key_row(g, w, ftab, fbias, head, kt * TM + tid, bias));
      kbias[tid] = bias;
    }
    __syncthreads();
    fill_split<false>(smem + Smem::K, ptr, 0);
    fill_split<false>(smem + Smem::V, ptr, g.C);
    fence_proxy_async_smem();
    __syncthreads();
    float s[32], p[32];
    wgmma_fence();
    mma_rows(s, sb + Smem::Q, sb + Smem::K);          // S = Q K^T
    mma_rows(p, sb + Smem::O, sb + Smem::V);          // dP = dO V^T
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float x[16], mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          x[2 * j + e] = fmaf(s[4 * j + 2 * h + e], g.scale_log2, kbias[8 * j + 2 * quad + e]);
          mx = fmaxf(mx, x[2 * j + e]);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[h], mx), alpha = exp2f(m[h] - mn);
      float ls = 0.f, as = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pe = exp2f(x[2 * j + e] - mn);
          ls += pe;
          as = fmaf(pe, p[4 * j + 2 * h + e], as);
        }
      ls += __shfl_xor_sync(0xffffffffu, ls, 1);
      ls += __shfl_xor_sync(0xffffffffu, ls, 2);
      as += __shfl_xor_sync(0xffffffffu, as, 1);
      as += __shfl_xor_sync(0xffffffffu, as, 2);
      l[h] = fmaf(l[h], alpha, ls);
      a[h] = fmaf(a[h], alpha, as);
      m[h] = mn;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qi = q0 + rw + 8 * h;
    if (qi < nq && quad == 0) {
      float* st = g.stats + ((static_cast<size_t>(bw) * g.heads + head) * nq + qi) * 2;
      st[0] = m[h] + log2f(l[h]);
      st[1] = a[h] / l[h];
    }
  }
}

// ------------------------------------------------------------------------------------------------------ 2. keys
__global__ void __launch_bounds__(THREADS, 1) attn_grad_keys_kernel(const __grid_constant__ Geo g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = aligned_smem(smem_raw);
  float* kbias = reinterpret_cast<float*>(smem + Smem::CB);
  float* qlse = reinterpret_cast<float*>(smem + Smem::CL);
  float* qD = reinterpret_cast<float*>(smem + Smem::CD);
  float* fbias = reinterpret_cast<float*>(smem + Smem::FB);
  int* ftab = reinterpret_cast<int*>(smem + Smem::FT);
  uint64_t* ptr = reinterpret_cast<uint64_t*>(smem + Smem::PTR);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = lane & 3;
  const int rw = 16 * warp + (lane >> 2);
  const int nW = g.nWh * g.nWw, grp = blockIdx.x;
  const int unit_local = blockIdx.z / nW, win = blockIdx.z % nW, unit = g.unit0 + unit_local;
  const int b = unit / g.heads, head = unit % g.heads, bw = b * nW + win;
  const Win w = make_win(g, b, win);
  const int nq = g.T * g.wh * g.ww, num_kt = (w.NK + TM - 1) / TM, num_qt = (nq + TM - 1) / TM;
  const size_t C3 = 3 * static_cast<size_t>(g.C);
  const uint32_t sb = smem_u32(smem);
  float* dqp = g.part_dq + ((static_cast<size_t>(unit_local) * nW + win) * GROUPS + grp) * nq * HD;
  const float* st = g.stats + (static_cast<size_t>(bw) * g.heads + head) * nq * 2;
  if (grp >= num_kt) {                                 // uniform: no key tile for this group, its dQ partial is 0
    for (int i = tid; i < nq * HD; i += THREADS) dqp[i] = 0.f;
    return;
  }

  build_frame_table(g, w, ftab, fbias);
  for (int kt = grp; kt < num_kt; kt += GROUPS) {
    __syncthreads();
    if (tid < TM) {
      float bias;
      ptr[tid] = reinterpret_cast<uint64_t>(key_row(g, w, ftab, fbias, head, kt * TM + tid, bias));
      kbias[tid] = bias;
    }
    __syncthreads();
    fill_split<false>(smem + Smem::K, ptr, 0);
    fill_split<false>(smem + Smem::V, ptr, g.C);
    const float rb[2] = {kbias[rw], kbias[rw + 8]};
    float dk[64], dv[64];
    for (int qt = 0; qt < num_qt; ++qt) {
      __syncthreads();                                 // the previous step's MMAs and reads of ptr / qlse / qD are done
      if (tid < TM) {
        const int qi = qt * TM + tid;
        const size_t tok = qi < nq ? query_token(g, w, qi) : 0;
        ptr[TM + tid] = qi < nq ? reinterpret_cast<uint64_t>(g.qkv + tok * C3 + head * HD) : 0;
        ptr[2 * TM + tid] = qi < nq ? reinterpret_cast<uint64_t>(g.dout + tok * g.C + head * HD) : 0;
        qlse[tid] = qi < nq ? st[2 * qi] : INFINITY;   // past the window's queries: P = 0
        qD[tid] = qi < nq ? st[2 * qi + 1] : 0.f;
      }
      __syncthreads();
      fill_split<false>(smem + Smem::Q, ptr + TM, 0);
      fill_split<true>(smem + Smem::O, ptr + 2 * TM, 0);
      fence_proxy_async_smem();
      __syncthreads();
      // ---- S^T = K Q^T, dP^T = V dO^T: rows = the tile's keys, columns = the tile's queries
      float s[32], p[32];
      wgmma_fence();
      mma_rows(s, sb + Smem::K, sb + Smem::Q);
      mma_rows(p, sb + Smem::V, sb + Smem::O);
      wgmma_commit();
      wgmma_wait<0>();
      // ---- P^T and dS^T = P^T (dP^T - D) -> shared memory as bf16 (hi, lo), [64 keys][64 queries]
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + 2 * quad;
        const float l0 = qlse[c], l1 = qlse[c + 1], d0 = qD[c], d1 = qD[c + 1];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float p0 = exp2f(fmaf(s[4 * j + 2 * h], g.scale_log2, rb[h]) - l0);
          const float p1 = exp2f(fmaf(s[4 * j + 2 * h + 1], g.scale_log2, rb[h]) - l1);
          const float ds0 = p0 * (p[4 * j + 2 * h] - d0), ds1 = p1 * (p[4 * j + 2 * h + 1] - d1);
          const uint32_t o = sw128_offset(rw + 8 * h, j) + 4 * quad;
          const __nv_bfloat162 ph = __floats2bfloat162_rn(p0, p1), dh = __floats2bfloat162_rn(ds0, ds1);
          const float2 phf = __bfloat1622float2(ph), dhf = __bfloat1622float2(dh);
          *reinterpret_cast<__nv_bfloat162*>(smem + Smem::P + o) = ph;
          *reinterpret_cast<__nv_bfloat162*>(smem + Smem::P + ATOM + o) = __floats2bfloat162_rn(p0 - phf.x, p1 - phf.y);
          *reinterpret_cast<__nv_bfloat162*>(smem + Smem::DS + o) = dh;
          *reinterpret_cast<__nv_bfloat162*>(smem + Smem::DS + ATOM + o) =
              __floats2bfloat162_rn(ds0 - dhf.x, ds1 - dhf.y);
        }
      }
      fence_proxy_async_smem();
      __syncthreads();
      // ---- dV += P^T dO, dK += dS^T Q (16 queries per k16 step); dQ_tile = dS K (16 keys per step)
      float dq[64];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TM / 16; ++k) {
        const uint32_t acc = (qt | k) != 0;
        const uint64_t ph = gmma_desc_sw128(sb + Smem::P, 16, 1024) + 2 * k, pl = ph + (ATOM >> 4);
        const uint64_t dh = gmma_desc_sw128(sb + Smem::DS, 16, 1024) + 2 * k, dl = dh + (ATOM >> 4);
        const uint64_t oh = mdesc(sb + Smem::O, k), ol = oh + (TILE >> 4);
        const uint64_t qh = mdesc(sb + Smem::Q, k), ql = qh + (TILE >> 4);
        wgmma_n128_bf16_tb(dv, pl, oh, acc);
        wgmma_n128_bf16_tb(dv, ph, ol, 1);
        wgmma_n128_bf16_tb(dv, ph, oh, 1);
        wgmma_n128_bf16_tb(dk, dl, qh, acc);
        wgmma_n128_bf16_tb(dk, dh, ql, 1);
        wgmma_n128_bf16_tb(dk, dh, qh, 1);
      }
#pragma unroll
      for (int k = 0; k < TM / 16; ++k) {
        const uint64_t ah = mdesc(sb + Smem::DS, k), al = ah + (ATOM >> 4);
        const uint64_t kh = mdesc(sb + Smem::K, k), kl = kh + (TILE >> 4);
        wgmma_n128_bf16_tt(dq, al, kh, k != 0);
        wgmma_n128_bf16_tt(dq, ah, kl, 1);
        wgmma_n128_bf16_tt(dq, ah, kh, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // ---- this group's dQ partial: written by its first key tile, then added to in key-tile order
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int qi = qt * TM + rw + 8 * h;
        if (qi >= nq) continue;
        float* d = dqp + static_cast<size_t>(qi) * HD;
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
          float2 v = make_float2(dq[4 * j + 2 * h] * g.scale, dq[4 * j + 2 * h + 1] * g.scale);
          float2* dst = reinterpret_cast<float2*>(d + 8 * j + 2 * quad);
          if (kt != grp) {
            const float2 o = *dst;
            v.x += o.x;
            v.y += o.y;
          }
          *dst = v;
        }
      }
    }
    // ---- dK | dV of the tile's key slots
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int kk = kt * TM + rw + 8 * h;
      if (kk >= w.NK) continue;
      float* dst = g.part + ((static_cast<size_t>(unit_local) * nW + win) * g.NKS + kk) * (2 * HD);
#pragma unroll
      for (int j = 0; j < HD / 8; ++j) {
        const int c = 8 * j + 2 * quad;
        *reinterpret_cast<float2*>(dst + c) = make_float2(dk[4 * j + 2 * h] * g.scale, dk[4 * j + 2 * h + 1] * g.scale);
        *reinterpret_cast<float2*>(dst + HD + c) = make_float2(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------ 3. gather
// blockIdx.x = key token of the clip (ring tokens (t, y, x), then pooled tokens (t, pi, pj)), blockIdx.y = unit in the
// chunk; thread d < 128: dK channel d, thread 128 + d: dV channel d
__global__ void __launch_bounds__(2 * HD) attn_grad_gather_kernel(const __grid_constant__ Geo g) {
  __shared__ int s_win[MAX_SOURCES], s_slot[MAX_SOURCES], s_mult[MAX_SOURCES], s_n;
  const int nW = g.nWh * g.nWw;
  const int unit_local = blockIdx.y, unit = g.unit0 + unit_local;
  const int b = unit / g.heads, head = unit % g.heads;
  const int ring_tokens = g.T * g.H * g.W;
  int tok = blockIdx.x;
  const int pooled = tok >= ring_tokens;
  if (pooled) tok -= ring_tokens;
  const int gw = pooled ? g.nWw : g.W, gh = pooled ? g.nWh : g.H;
  const int t = tok / (gh * gw), y = (tok / gw) % gh, x = tok % gw;
  if (threadIdx.x == 0) s_n = key_sources(g, t, pooled, y, x, s_win, s_slot, s_mult, MAX_SOURCES);
  __syncthreads();
  float acc = 0.f;
  const float* part = g.part + static_cast<size_t>(unit_local) * nW * g.NKS * (2 * HD) + threadIdx.x;
  for (int i = 0; i < s_n; ++i) acc += part[(static_cast<size_t>(s_win[i]) * g.NKS + s_slot[i]) * (2 * HD)];
  const size_t C3 = 3 * static_cast<size_t>(g.C);
  const size_t row = static_cast<size_t>(b) * g.T * gh * gw + tok;
  float* dst = (pooled ? g.dpooled : g.dqkv) + row * C3 + head * HD;
  dst[(threadIdx.x < HD ? g.C : 2 * g.C - HD) + threadIdx.x] = acc;   // dK channel d, or dV channel d - 128
  if (threadIdx.x >= HD) return;
  if (pooled) {
    dst[threadIdx.x] = 0.f;                            // the pooled rows' q is never read
    return;
  }
  // dQ of the token: the query (t, y % wh, x % ww) of window (y / wh, x / ww), its groups' partials in order
  const int win = (y / g.wh) * g.nWw + x / g.ww, nq = g.T * g.wh * g.ww;
  const int qi = t * g.wh * g.ww + (y % g.wh) * g.ww + x % g.ww;
  const float* dqp = g.part_dq + (static_cast<size_t>(unit_local) * nW + win) * GROUPS * nq * HD + qi * HD + threadIdx.x;
  float dq = 0.f;
  for (int grp = 0; grp < GROUPS; ++grp) dq += dqp[static_cast<size_t>(grp) * nq * HD];
  dst[threadIdx.x] = dq;
}

// host side -------------------------------------------------------------------------------------------------------
static int make_geo(Geo& g, int b, int t, int h, int w, int heads, int wh, int ww, int eh, int ew, int fh, int fw,
                    int use_pooled, float scale) {
  const int EH = wh + 2 * eh, EW = ww + 2 * ew;
  if (EH * EW > MAX_RING || EH * EW + (use_pooled ? fh * fw : 0) > MAX_FRAME_KEYS) {
    set_error("focal attention backward: expanded window %dx%d (+%dx%d pooled) exceeds the per-frame key table", EH, EW,
              fh, fw);
    return -2;
  }
  if ((EH / wh + 2) * (EW / ww + 2) > MAX_SOURCES || (use_pooled && fh * fw > MAX_SOURCES)) {
    set_error("focal attention backward: a key token reaches more than %d (window, key) pairs", MAX_SOURCES);
    return -2;
  }
  if (static_cast<long long>(h) * w * 3 * heads * HD > 0x7FFFFFFFLL) {
    set_error("focal attention backward: one frame of qkv exceeds 2^31 elements");
    return -2;
  }
  g = Geo{};
  g.B = b; g.T = t; g.H = h; g.W = w; g.heads = heads; g.C = heads * HD;
  g.wh = wh; g.ww = ww; g.eh = eh; g.ew = ew; g.fh = fh; g.fw = fw;
  g.nWh = h / wh; g.nWw = w / ww;
  g.use_pooled = use_pooled;
  g.scale = scale;
  g.scale_log2 = scale * LOG2E;
  attn::order_ring(wh, ww, eh, ew, g.ring_pos, g.ring_mult, g.n1, g.n2);
  for (int e = 0; e < MAX_RING; ++e) g.ring_slot[e] = 255;
  for (int s = 0; s < g.n1 + g.n2; ++s) g.ring_slot[g.ring_pos[s]] = static_cast<uint8_t>(s);
  g.NKS = t * (g.n1 + g.n2 + (use_pooled ? fh * fw : 0));
  return 0;
}

static long long stats_elems(const Geo& g) {
  return (static_cast<long long>(g.B) * g.nWh * g.nWw * g.heads * g.T * g.wh * g.ww * 2 + 3) / 4 * 4;
}
static long long unit_kv_elems(const Geo& g) { return static_cast<long long>(g.nWh) * g.nWw * g.NKS * 2 * HD; }
static long long unit_elems(const Geo& g) {
  return unit_kv_elems(g) + static_cast<long long>(g.nWh) * g.nWw * GROUPS * g.T * g.wh * g.ww * HD;
}
static int units_per_chunk(const Geo& g) {
  const long long units = static_cast<long long>(g.B) * g.heads;
  long long n = PARTIAL_BUDGET / unit_elems(g);
  n = n < 1 ? 1 : n;
  return static_cast<int>(n < units ? n : units);
}

}  // namespace attn_grad

long long focal_attention_backward_work_elems(int b, int t, int h, int w, int heads, int wh, int ww, int eh, int ew,
                                              int fh, int fw, int use_pooled) {
  using namespace attn_grad;
  Geo g;
  if (const int e = make_geo(g, b, t, h, w, heads, wh, ww, eh, ew, fh, fw, use_pooled, 1.f)) return e;
  if (b == 0) return 0;
  return stats_elems(g) + units_per_chunk(g) * unit_elems(g);
}

int focal_attention_key_sources(int t_count, int h, int w, int wh, int ww, int eh, int ew, int fh, int fw,
                                int use_pooled, int t, int pooled, int y, int x, int* win, int* slot, int* mult, int cap) {
  using namespace attn_grad;
  Geo g;
  if (const int e = make_geo(g, 1, t_count, h, w, 1, wh, ww, eh, ew, fh, fw, use_pooled, 1.f)) return e;
  return key_sources(g, t, pooled, y, x, win, slot, mult, cap);
}

int launch_focal_attention_backward(const void* qkv, const void* qkv_pooled, const float* dout, float* dqkv,
                                    float* dqkv_pooled, float* work, int b, int t, int h, int w, int heads, int wh,
                                    int ww, int eh, int ew, int fh, int fw, int use_pooled, float scale,
                                    cudaStream_t stream) {
  using namespace attn_grad;
  Geo g;
  if (const int e = make_geo(g, b, t, h, w, heads, wh, ww, eh, ew, fh, fw, use_pooled, scale)) return e;
  if (b == 0) return 0;
  g.qkv = static_cast<const __half*>(qkv);
  g.pooled = static_cast<const __half*>(qkv_pooled);
  g.dout = dout;
  g.dqkv = dqkv;
  g.dpooled = dqkv_pooled;
  g.stats = work;
  g.part = work + stats_elems(g);
  const int nW = g.nWh * g.nWw;
  const long long nwin = static_cast<long long>(b) * nW;
  const int chunk = units_per_chunk(g);
  g.part_dq = g.part + chunk * unit_kv_elems(g);
  if (nwin > 65535 || static_cast<long long>(chunk) * nW > 65535 || heads > 65535) {
    set_error("focal attention backward: grid too large (B*nW=%lld)", nwin);
    return -2;
  }
  static DeviceOnce cfg;
  if (const int e = configure_once(cfg, SMEM_BYTES, attn_grad_rows_kernel, attn_grad_keys_kernel)) return e;
  const int nq = t * wh * ww;
  attn_grad_rows_kernel<<<dim3((nq + TM - 1) / TM, heads, static_cast<unsigned>(nwin)), THREADS, SMEM_BYTES, stream>>>(g);
  count_launch();
  const int units = b * heads;
  const unsigned tokens = static_cast<unsigned>(t * h * w + (use_pooled ? t * nW : 0));
  for (int u0 = 0; u0 < units; u0 += chunk) {
    g.unit0 = u0;
    const int n = units - u0 < chunk ? units - u0 : chunk;
    attn_grad_keys_kernel<<<dim3(GROUPS, 1, n * nW), THREADS, SMEM_BYTES, stream>>>(g);
    count_launch();
    attn_grad_gather_kernel<<<dim3(tokens, n), 2 * HD, 0, stream>>>(g);
    count_launch();
  }
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
