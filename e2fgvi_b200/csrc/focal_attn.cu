// Temporal focal window attention core — replaces model/modules/tfocal_transformer.py:226-396 (+ window_reverse
// :528): softmax(q k_all^T) v_all per (window, head) with k_all = own window | 4 circularly rolled ring sets |
// pooled-window neighbourhood, without materialising rolled copies, the key list or the logits.
//
// Key set per (window (wi,wj), frame t), equivalent to the reference's list (order is irrelevant to softmax.V):
//   * the expanded window (wh+2eh) x (ww+2ew) around the query window, coordinates wrapped modulo (H, W) exactly
//     like torch.roll; a token listed m times by the reference (own window + tl/tr/bl/br rolls after
//     valid_ind_rolled; m = 2 for the 12 duplicated ring tokens) gets log2(m) added to its log2-domain logit;
//   * the in-grid pooled windows of the (fh x fw) neighbourhood; zero-padded neighbours have k = v = 0 and a -100
//     logit in the reference (:301-316, :377-380): they only add n_masked * exp(-100) to the softmax denominator,
//     which is folded into the initial (running max, running sum) = (-100, n_masked).
//   Keys are ordered [multiplicity-1 ring keys | pooled keys | multiplicity>=2 ring keys | padding], so only the
//   last key tile(s) carry a non-zero logit bias and every other tile takes a bias-free fast path.
//
// One CTA = one (128-query tile, head, window).
// Warp roles (384 threads):
//   warps 0-7  two softmax warpgroups, 64 query rows each: S = Q K^T by wgmma (Q, K K-major in smem) into registers,
//              online softmax with lazy rescale on the accumulator fragment (a row lives in the 4 threads of a quad),
//              P packed to fp16 IN REGISTERS as the A operand of O += P V (wgmma, V an MN-major B operand in smem) —
//              no P tile in shared memory; final O / l -> global (un-partitioned layout)
//   warps 8-11 loaders: per-key source addresses (wrap / pooled / padding) then coalesced 16-byte cp.async gathers of
//              K and V rows (256 B each) into swizzled smem, 2-stage ring of 64-key tiles
// Roofline (SURVEY §8d): 4*B*nW*heads*(T*wh*ww)*(T*(wh*ww+ring+fh*fw))*128 FLOP on the tensor pipe.
#include <type_traits>
#include <cuda_bf16.h>
#include "common.cuh"
#include "focal_geom.cuh"
#include "launch.h"

namespace e2f {
namespace attn {

constexpr int HD = 128;                    // head dim
constexpr int BM = 128, BN = 64;           // query tile, key tile
constexpr int QATOM = BM * 128;            // [128 rows][64 halfs] swizzled sub-tile of Q
constexpr int KATOM = BN * 128;            // [64 keys][64 halfs] swizzled sub-tile of K / V
constexpr int QTILE = 2 * QATOM;           // 32 KB
constexpr int KTILE = 2 * KATOM;           // 16 KB
constexpr int KV_STAGES = 2;
constexpr int BIAS_SLOTS = 4;              // logit-bias rows outlive their K stage (the K stage is recycled after S, not PV)
constexpr int SOFTMAX_WARPS = 8, LOADER_WARPS = 4;
constexpr int SOFTMAX_THREADS = SOFTMAX_WARPS * 32;
constexpr int THREADS = (SOFTMAX_WARPS + LOADER_WARPS) * 32;   // 384
constexpr float LOG2E = 1.4426950408889634f;
constexpr float RESCALE_THRESHOLD = 8.0f;      // log2 domain: P stays <= 2^8
constexpr int MAX_FRAME_KEYS = 384;            // ring + pooled keys of one frame (198 for 5x9 / 5x9)

struct Smem {
  static constexpr int Q = 0;
  static constexpr int K = Q + QTILE;
  static constexpr int V = K + KV_STAGES * KTILE;
  static constexpr int KEYPTR = V + KV_STAGES * KTILE;          // [128] uint64 (Q rows at start, then [stages][64])
  static constexpr int BIAS = KEYPTR + BM * 8;                  // [BIAS_SLOTS][64] float (slot = key tile & 3)
  static constexpr int FTAB = BIAS + BIAS_SLOTS * BN * 4;       // [MAX_FRAME_KEYS] int32: key offset inside its frame
  static constexpr int FBIAS = FTAB + MAX_FRAME_KEYS * 4;       // [MAX_FRAME_KEYS] float: logit bias (log2 multiplicity)
  static constexpr int BARS = FBIAS + MAX_FRAME_KEYS * 4;
  static constexpr int NUM_BARS = 1 + 4 * KV_STAGES;
  static constexpr int BYTES = BARS + NUM_BARS * 8;
};
constexpr int SMEM_BYTES = Smem::BYTES + 1024;

struct Params {
  const __half* qkv;
  const __half* pooled;
  void* out;
  void* out_lo;                   // E2F_SPLIT_BF16 only: low term, [B][T][H][W][C] bf16 right behind the high term
  int B, T, H, W, heads, C;       // C = heads*128
  int wh, ww, eh, ew, fh, fw;
  int nWh, nWw;
  int use_pooled;
  float scale_log2;               // scale * log2(e)
  int n1, n2;                     // expanded-window positions listed once / more than once by the reference
  uint8_t ring_pos[MAX_RING];     // positions (er*EW + ec): the n1 single ones first, then the n2 multiple ones
  uint8_t ring_mult[MAX_RING];    // multiplicity of each entry
};

__device__ __forceinline__ void loader_barrier() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// coalesced gather of ROWS rows x 256 B (two 64-half atoms of ROWS*128 B) into a swizzled tile; 16 lanes cover one
// row, the 4 loader warps split the rows.
template <int ROWS>
__device__ __forceinline__ void gather_rows(uint32_t tile_smem, const uint64_t* row_ptr, int lwarp, int lane,
                                            int half_offset) {
  const int chunk = lane & 15;
  const uint32_t atom_off = (chunk >> 3) * (ROWS * 128);
#pragma unroll 4
  for (int it = 0; it < ROWS / 8; ++it) {
    const int row = lwarp * (ROWS / 4) + it * 2 + (lane >> 4);
    uint64_t p;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(p) : "r"(smem_u32(row_ptr + row)));
    const uint32_t dst = tile_smem + atom_off + sw128_offset(row, chunk & 7);
    const __half* src = reinterpret_cast<const __half*>(p) + half_offset + chunk * 8;
    cp_async16_zfill(dst, p ? static_cast<const void*>(src) : static_cast<const void*>(row_ptr), p ? 16u : 0u);
  }
}

struct SplitBf16 {                // output tag: bf16 (hi, lo) two-term split of the result (operand of e2f_linear_bf16x3)
  __nv_bfloat16 v;
};

template <typename OutT>
__global__ void __launch_bounds__(THREADS, 1) focal_attn_kernel(const __grid_constant__ Params prm) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* key_ptr = reinterpret_cast<uint64_t*>(smem + Smem::KEYPTR);
  float* key_bias = reinterpret_cast<float*>(smem + Smem::BIAS);
  int* ftab = reinterpret_cast<int*>(smem + Smem::FTAB);
  float* fbias = reinterpret_cast<float*>(smem + Smem::FBIAS);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Smem::BARS);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;
  uint64_t* v_full = k_full + KV_STAGES;
  uint64_t* k_empty = v_full + KV_STAGES;       // K stage read by S(kt): free again as soon as that MMA completes
  uint64_t* v_empty = k_empty + KV_STAGES;      // V stage read by PV(kt)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- problem geometry (uniform per CTA)
  const int area = prm.wh * prm.ww;
  const int nq = prm.T * area;
  const int qt = blockIdx.x, head = blockIdx.y;
  const int win = blockIdx.z % (prm.nWh * prm.nWw), b = blockIdx.z / (prm.nWh * prm.nWw);
  const int wi = win / prm.nWw, wj = win % prm.nWw;
  const int EW = prm.ww + 2 * prm.ew;
  int pi0 = 0, pj0 = 0, PH = 0, PW = 0;
  if (prm.use_pooled) {
    pi0 = max(0, wi - prm.fh / 2);
    pj0 = max(0, wj - prm.fw / 2);
    PH = min(prm.nWh - 1, wi + prm.fh / 2) - pi0 + 1;
    PW = min(prm.nWw - 1, wj + prm.fw / 2) - pj0 + 1;
  }
  const int npool = PH * PW;
  const int n_masked = prm.use_pooled ? prm.T * (prm.fh * prm.fw - npool) : 0;
  const int nA = prm.T * prm.n1;                 // single-listed ring keys (bias 0)
  const int nB = nA + prm.T * npool;             // + pooled keys (bias 0)
  const int NK = nB + prm.T * prm.n2;            // + multiply-listed ring keys (bias log2 m)
  const int num_kt = (NK + BN - 1) / BN;
  // first key tile that may contain a non-zero bias (multiplicity keys or -inf padding)
  const int bias_kt = (NK % BN) ? min(nB / BN, num_kt - 1) : ((prm.n2 > 0) ? nB / BN : num_kt);
  const size_t C3 = 3 * static_cast<size_t>(prm.C);

  if (tid == 0) {
    mbar_init(q_full, LOADER_WARPS);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(&k_full[s], LOADER_WARPS);
      mbar_init(&v_full[s], LOADER_WARPS);
      mbar_init(&k_empty[s], SOFTMAX_WARPS);
      mbar_init(&v_empty[s], SOFTMAX_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < SOFTMAX_WARPS) {
    // =================================================================== softmax + epilogue
    // accumulator fragments (common.cuh): this thread holds rows rw and rw + 8 of its warpgroup's 64 query rows, key /
    // channel column pairs 8j + 2(lane % 4); the 4 threads of a quad share a row
    const int wg = warp >> 2, wq = warp & 3, quad = lane & 3;
    const int rw = wg * 64 + wq * 16 + (lane >> 2);
    float m_used[2], l[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      m_used[h] = n_masked > 0 ? -100.0f * LOG2E : -INFINITY;
      l[h] = quad == 0 ? static_cast<float>(n_masked) : 0.f;     // partial row sums, reduced over the quad at the end
    }
    const float sc = prm.scale_log2;
    const uint64_t dq0 = gmma_desc_sw128(smem_u32(smem + Smem::Q) + wg * 64 * 128, 16, 1024);
    const uint64_t dq1 = gmma_desc_adv(dq0, QATOM);
    const uint64_t dk0 = gmma_desc_sw128(smem_u32(smem + Smem::K), 16, 1024);
    const uint64_t dv0 = gmma_desc_sw128(smem_u32(smem + Smem::V), KATOM, 1024);
    float o[HD / 2];
    mbar_wait(q_full, 0);

    for (int kt = 0; kt < num_kt; ++kt) {
      const int stage = kt % KV_STAGES;
      const bool biased = kt >= bias_kt;                // uniform over the CTA
      mbar_wait(&k_full[stage], (kt / KV_STAGES) & 1);
      // ---- S = Q K^T (64 rows x 64 keys per warpgroup)
      float s[BN / 2];
      const uint64_t dk = dk0 + ((stage * KTILE) >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k)
        wgmma_ss<64, true>(s, (k < 4 ? dq0 : dq1) + 2 * (k & 3), dk + (k < 4 ? 0 : (KATOM >> 4)) + 2 * (k & 3), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[stage]);      // S(kt) was the only reader of this K stage

      // ---- online softmax, log2 domain
      const float* kb = key_bias + (kt & (BIAS_SLOTS - 1)) * BN;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * quad;
        const float b0 = biased ? kb[c] : 0.f, b1 = biased ? kb[c + 1] : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float a0 = s[4 * j + 2 * h], a1 = s[4 * j + 2 * h + 1];
          if (biased) {
            a0 = fmaf(a0, sc, b0);
            a1 = fmaf(a1, sc, b1);
          }
          mx[h] = fmaxf(mx[h], fmaxf(a0, a1));
        }
      }
      float neg_m[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        if (!biased) mx[h] *= sc;                        // scale > 0: max commutes with the scaling
        // lazy rescale: only move the reference max when it grew by more than 2^8
        if (m_used[h] == -INFINITY) {
          m_used[h] = mx[h];                             // first tile without masked keys: nothing accumulated yet
        } else if (mx[h] - m_used[h] > RESCALE_THRESHOLD) {
          const float alpha = fast_exp2(m_used[h] - mx[h]);
          m_used[h] = mx[h];
          l[h] *= alpha;
          if (kt > 0) {
#pragma unroll
            for (int j = 0; j < HD / 8; ++j) {
              o[4 * j + 2 * h] *= alpha;
              o[4 * j + 2 * h + 1] *= alpha;
            }
          }
        }
        neg_m[h] = -m_used[h];
      }
      // P = exp2(s - m) packed to fp16: pk[j][h] = keys 8j + 2(lane % 4) + {0, 1} of row h, which is exactly the
      // register A fragment of the next MMA (k step kk takes j = 2kk and 2kk + 1)
      uint32_t pk[BN / 8][2];
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * quad;
        const float b0 = biased ? kb[c] : 0.f, b1 = biased ? kb[c + 1] : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float a0 = s[4 * j + 2 * h], a1 = s[4 * j + 2 * h + 1];
          if (biased) {
            a0 = fmaf(a0, sc, b0) + neg_m[h];
            a1 = fmaf(a1, sc, b1) + neg_m[h];
          } else {
            a0 = fmaf(a0, sc, neg_m[h]);
            a1 = fmaf(a1, sc, neg_m[h]);
          }
          const float p0 = fast_exp2(a0), p1 = fast_exp2(a1);
          l[h] += p0 + p1;
          pk[j][h] = pack_half2(p0, p1);
        }
      }

      // ---- O += P V
      mbar_wait(&v_full[stage], (kt / KV_STAGES) & 1);
      const uint64_t dv = dv0 + ((stage * KTILE) >> 4);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        const uint32_t a[4] = {pk[2 * kk][0], pk[2 * kk][1], pk[2 * kk + 1][0], pk[2 * kk + 1][1]};
        const uint64_t bdesc = dv + kk * (2048 >> 4);    // 16 keys = two 8-key groups of 1024 B
        const uint32_t acc = (kt | kk) != 0;
        wgmma_n64_f16_rs_tb(o, a, bdesc, acc);                        // channels [0, 64)
        wgmma_n64_f16_rs_tb(o + 32, a, bdesc + (KATOM >> 4), acc);    // channels [64, 128)
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[stage]);
    }

    // ---- epilogue: O / l -> out[b, t, y, x, head*128 ..]
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      const int qi = qt * BM + rw + 8 * h;
      if (qi >= nq) continue;
      const float inv_l = 1.0f / l[h];
      const int t = qi / area, p = qi - t * area;
      const int y = wi * prm.wh + p / prm.ww, x = wj * prm.ww + p % prm.ww;
      const size_t tok = ((static_cast<size_t>(b) * prm.T + t) * prm.H + y) * prm.W + x;
      const size_t dst_off = tok * prm.C + head * HD;
#pragma unroll
      for (int j = 0; j < HD / 8; ++j) {
        const size_t e = dst_off + 8 * j + 2 * quad;
        const float f0 = o[4 * j + 2 * h] * inv_l, f1 = o[4 * j + 2 * h + 1] * inv_l;
        if constexpr (std::is_same<OutT, SplitBf16>::value) {
          const __nv_bfloat162 hb = __floats2bfloat162_rn(f0, f1);
          const float2 hf = __bfloat1622float2(hb);
          *reinterpret_cast<__nv_bfloat162*>(static_cast<__nv_bfloat16*>(prm.out) + e) = hb;
          *reinterpret_cast<__nv_bfloat162*>(static_cast<__nv_bfloat16*>(prm.out_lo) + e) =
              __floats2bfloat162_rn(f0 - hf.x, f1 - hf.y);
        } else if constexpr (sizeof(OutT) == 4) {
          *reinterpret_cast<float2*>(static_cast<float*>(prm.out) + e) = make_float2(f0, f1);
        } else {
          *reinterpret_cast<uint32_t*>(static_cast<__half*>(prm.out) + e) = pack_half2(f0, f1);
        }
      }
    }
  } else {
    // =================================================================== loaders
    const int lt = tid - SOFTMAX_THREADS;               // 0..127
    const int lwarp = lt >> 5;
    // Q tile: row lt's source address (key_ptr is borrowed as scratch before the first K tile)
    {
      const int qi = qt * BM + lt;
      uint64_t p = 0;
      if (qi < nq) {
        const int t = qi / area, pp = qi - t * area;
        const int y = wi * prm.wh + pp / prm.ww, x = wj * prm.ww + pp % prm.ww;
        const size_t tok = ((static_cast<size_t>(b) * prm.T + t) * prm.H + y) * prm.W + x;
        p = reinterpret_cast<uint64_t>(prm.qkv + tok * C3 + head * HD);
      }
      key_ptr[lt] = p;
      loader_barrier();
      gather_rows<BM>(smem_u32(smem + Smem::Q), key_ptr, lwarp, lane, 0);
      cp_async_commit();
      cp_async_wait<0>();
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(q_full);
      loader_barrier();                                 // everyone done reading key_ptr[0..127]
    }
    // ---- per-frame key table, built once per CTA: entry e -> offset (in halfs) of that key's token inside its frame
    //      and its logit bias; entries ordered [n1 single ring | npool pooled | n2 multiple ring]
    const int nf = prm.n1 + npool + prm.n2;
    for (int e = lt; e < nf; e += LOADER_WARPS * 32) {
      int off;
      float bias = 0.f;
      if (e >= prm.n1 && e < prm.n1 + npool) {
        const int pp = e - prm.n1;
        off = ((pi0 + pp / PW) * prm.nWw + (pj0 + pp % PW)) * static_cast<int>(C3);
      } else {
        const int slot = (e < prm.n1) ? e : e - npool;
        const int pos = prm.ring_pos[slot], mult = prm.ring_mult[slot];
        const int er = pos / EW, ec = pos - er * EW;
        int y = (wi * prm.wh - prm.eh + er) % prm.H;
        int x = (wj * prm.ww - prm.ew + ec) % prm.W;
        y += (y < 0) ? prm.H : 0;
        x += (x < 0) ? prm.W : 0;
        off = (y * prm.W + x) * static_cast<int>(C3);
        bias = (mult == 1) ? 0.f : log2f(static_cast<float>(mult));
      }
      ftab[e] = off;
      fbias[e] = bias;
    }
    loader_barrier();
    const size_t ring_frame = static_cast<size_t>(prm.H) * prm.W * C3;
    const size_t pool_frame = static_cast<size_t>(prm.nWh) * prm.nWw * C3;
    const __half* ring_base = prm.qkv + static_cast<size_t>(b) * prm.T * ring_frame + prm.C + head * HD;
    const __half* pool_base = prm.pooled + static_cast<size_t>(b) * prm.T * pool_frame + prm.C + head * HD;
    for (int kt = 0; kt < num_kt; ++kt) {
      const int stage = kt % KV_STAGES;
      // ---- threads 0..63: address and logit bias of key (kt*64 + lt): (frame, entry) -> table lookup; computed
      //      BEFORE waiting for the stage to drain, so it is off the critical path
      uint64_t p = 0;
      float bias = -INFINITY;
      if (lt < BN) {
        const int idx = kt * BN + lt;
        if (idx < nA) {
          const int t = idx / prm.n1, e = idx - t * prm.n1;
          p = reinterpret_cast<uint64_t>(ring_base + t * ring_frame + ftab[e]);
          bias = 0.f;
        } else if (idx < nB) {
          const int j = idx - nA;
          const int t = j / npool, e = prm.n1 + (j - t * npool);
          p = reinterpret_cast<uint64_t>(pool_base + t * pool_frame + ftab[e]);
          bias = 0.f;
        } else if (idx < NK) {
          const int j = idx - nB;
          const int t = j / prm.n2, e = prm.n1 + npool + (j - t * prm.n2);
          p = reinterpret_cast<uint64_t>(ring_base + t * ring_frame + ftab[e]);
          bias = fbias[e];
        }
      }
      // The K stage is recycled as soon as S(kt-2) has read it (k_empty), the V stage only after PV(kt-2) (v_empty): the
      // gather of K(kt) — the operand the next S waits for — overlaps the softmax and the PV of the tiles in flight
      // instead of starting after them.
      mbar_wait(&k_empty[stage], ((kt / KV_STAGES) & 1) ^ 1);
      if (lt < BN) {
        key_ptr[stage * BN + lt] = p;
        key_bias[(kt & (BIAS_SLOTS - 1)) * BN + lt] = bias;
      }
      loader_barrier();
      gather_rows<BN>(smem_u32(smem + Smem::K + stage * KTILE), key_ptr + stage * BN, lwarp, lane, 0);
      cp_async_commit();
      if (kt > 0) {                                      // V(kt-1), committed one group earlier, has landed
        cp_async_wait<1>();
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_full[(kt - 1) % KV_STAGES]);
      }
      cp_async_wait<0>();                               // K landed
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_full[stage]);
      mbar_wait(&v_empty[stage], ((kt / KV_STAGES) & 1) ^ 1);
      gather_rows<BN>(smem_u32(smem + Smem::V + stage * KTILE), key_ptr + stage * BN, lwarp, lane, prm.C);
      cp_async_commit();
    }
    cp_async_wait<0>();                                 // V of the last tile
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_full[(num_kt - 1) % KV_STAGES]);
  }
}

}  // namespace attn

int launch_focal_attention(const void* qkv, const void* qkv_pooled, void* out, int b, int t, int h, int w, int heads,
                           int head_dim, int wh, int ww, int eh, int ew, int fh, int fw, int use_pooled, float scale,
                           int out_dtype, cudaStream_t stream) {
  using namespace attn;
  if (head_dim != HD) {
    set_error("focal attention: head_dim %d unsupported", head_dim);
    return -2;
  }
  if (b == 0) return 0;
  const int EH = wh + 2 * eh, EW = ww + 2 * ew;
  if (EH * EW > MAX_RING || EH * EW + (use_pooled ? fh * fw : 0) > MAX_FRAME_KEYS) {
    set_error("focal attention: expanded window %dx%d (+%dx%d pooled) exceeds the per-frame key table", EH, EW, fh, fw);
    return -2;
  }
  if (static_cast<long long>(h) * w * 3 * heads * HD > 0x7FFFFFFFLL) {
    set_error("focal attention: one frame of qkv exceeds 2^31 elements");
    return -2;
  }
  if (!(scale > 0.f)) {
    set_error("focal attention: scale must be positive");
    return -1;
  }
  Params prm;
  prm.qkv = static_cast<const __half*>(qkv);
  prm.pooled = static_cast<const __half*>(qkv_pooled);
  prm.out = out;
  prm.B = b; prm.T = t; prm.H = h; prm.W = w; prm.heads = heads; prm.C = heads * HD;
  prm.wh = wh; prm.ww = ww; prm.eh = eh; prm.ew = ew; prm.fh = fh; prm.fw = fw;
  prm.nWh = h / wh; prm.nWw = w / ww;
  prm.use_pooled = use_pooled;
  prm.scale_log2 = scale * LOG2E;
  // order the expanded-window positions: single-listed first, multiply-listed last (positions never listed are dropped)
  order_ring(wh, ww, eh, ew, prm.ring_pos, prm.ring_mult, prm.n1, prm.n2);
  const long long nwin = static_cast<long long>(b) * prm.nWh * prm.nWw;
  if (nwin > 65535 || heads > 65535) {
    set_error("focal attention: grid too large (B*nW=%lld)", nwin);
    return -2;
  }
  const dim3 grid((t * wh * ww + BM - 1) / BM, heads, static_cast<unsigned>(nwin));
  prm.out_lo = nullptr;
  static DeviceOnce cfg;
  if (const int e = configure_once_carveout(cfg, SMEM_BYTES, 100, focal_attn_kernel<SplitBf16>, focal_attn_kernel<__half>,
                                            focal_attn_kernel<float>))
    return e;
  if (out_dtype == 2) {
    prm.out_lo = static_cast<__nv_bfloat16*>(prm.out) + static_cast<size_t>(b) * t * h * w * prm.C;
    focal_attn_kernel<SplitBf16><<<grid, THREADS, SMEM_BYTES, stream>>>(prm);
  } else if (out_dtype == 1) {
    focal_attn_kernel<__half><<<grid, THREADS, SMEM_BYTES, stream>>>(prm);
  } else {
    focal_attn_kernel<float><<<grid, THREADS, SMEM_BYTES, stream>>>(prm);
  }
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace e2f
