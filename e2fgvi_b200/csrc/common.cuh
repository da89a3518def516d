// Hopper (sm_90a) device primitives used by every kernel in this library:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with shared-memory descriptors, fp32 accumulators in
// registers), cp.async, and small math helpers.  Everything is inline PTX; no CUTLASS dependency.  Bit layouts of
// the descriptors follow the PTX ISA "wgmma matrix descriptor" table.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>

namespace e2f {

#ifndef E2F_WAIT_LIMIT_NS
// A lost arrive must end in a trap (launch failure), never in a hung GPU: every 1024 polls the waiting thread reads
// %globaltimer and traps once a single wait has lasted E2F_WAIT_LIMIT_NS (a healthy wait takes microseconds to a few
// milliseconds).  Time-based, so the bound does not depend on how long one try_wait poll suspends in hardware.
#define E2F_WAIT_LIMIT_NS 20000000000ull
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      // suspend-time hint (ns): the waiting thread SLEEPS in hardware until the phase completes instead of
      // returning immediately — without it every waiting warp busy-polls and starves the working warps of
      // issue slots
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // bare poll loop: waiting warps share an SM sub-partition with working warps, so the loop body must stay tiny
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 1023u) == 0) {
      uint64_t now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > E2F_WAIT_LIMIT_NS) asm volatile("trap;");
    }
  }
}

// ----------------------------------------------------------------------------- proxies / fences
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------- cp.async (LDGSTS)
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
// src_bytes = 0 -> zero fill (no global read is performed)
__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor, 128-byte swizzle, 16-bit elements.
//   bits [0,14)  start address >> 4        bits [16,30) leading-dim byte offset >> 4
//   bits [32,46) stride-dim byte offset >> 4   bits [62,64) layout type: 1 = SWIZZLE_128B
// K-major tile  [rows][64 halfs]: rows are 128 B, 8-row groups are 1024 B apart (SBO); LBO unused (=1).
// MN-major tile [k][64 halfs]   : k-rows are 128 B, 8-k groups are SBO apart, the next 64 MN elements are LBO apart.
// The swizzle is a function of the absolute shared-memory address, so a start address moved by whole 128-byte rows
// (or by 32 bytes along K inside a row) addresses the same swizzled data: descriptors advance by one 64-bit add.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ uint64_t gmma_desc_adv(uint64_t desc, uint32_t bytes) { return desc + (bytes >> 4); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x n] (+)= A[64 x 16] . B[n x 16]^T, A and B K-major in shared memory, issued by a whole warpgroup.  Accumulator
// fragment of thread t (warp w = (t / 32) % 4, lane l): d[4j + {0,1}] = row 16w + l/4, columns 8j + 2(l%4) + {0,1};
// d[4j + {2,3}] = the same columns of row 16w + l/4 + 8.  acc = 0 overwrites D.
__device__ __forceinline__ void wgmma_n16_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_n16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_n32_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_n32_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_n64_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_n64_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_n64_f16_rs_tb(float* d, const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
}

// n = N (multiple of 16) as blocks of 64 / 32 / 16 columns; the B rows of the next block start n*128 bytes further
template <int N, bool F16>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  static_assert(N % 16 == 0 && N > 0, "wgmma N");
  if constexpr (N >= 64) {
    if constexpr (F16) wgmma_n64_f16(d, adesc, bdesc, acc);
    else wgmma_n64_bf16(d, adesc, bdesc, acc);
    if constexpr (N > 64) wgmma_ss<N - 64, F16>(d + 32, adesc, gmma_desc_adv(bdesc, 64 * 128), acc);
  } else if constexpr (N >= 32) {
    if constexpr (F16) wgmma_n32_f16(d, adesc, bdesc, acc);
    else wgmma_n32_bf16(d, adesc, bdesc, acc);
    if constexpr (N > 32) wgmma_ss<N - 32, F16>(d + 16, adesc, gmma_desc_adv(bdesc, 32 * 128), acc);
  } else {
    if constexpr (F16) wgmma_n16_f16(d, adesc, bdesc, acc);
    else wgmma_n16_bf16(d, adesc, bdesc, acc);
  }
}

// Accumulator staging: a warpgroup's fragments written to a [rows][N] fp32 shared-memory tile so that a thread can
// read a whole row (the row-per-thread epilogues).  16-byte chunk c of row r sits at chunk c ^ (r & 7): row-parallel
// 16-byte reads by 8 consecutive rows hit 8 different bank groups.
__device__ __forceinline__ uint32_t acc_stage_offset(uint32_t row, uint32_t col, uint32_t n) {
  return row * n * 4u + ((((col >> 2) ^ (row & 7u))) << 4) + (col & 3u) * 4u;
}
template <int N>
__device__ __forceinline__ void acc_stage_store(uint32_t stage_smem, const float* d, int row0, int lane) {
  // row0: first row of the calling warp's 16-row slice
  const int r = row0 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_smem + acc_stage_offset(r, 8 * j + c, N)),
                 "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_smem + acc_stage_offset(r + 8, 8 * j + c, N)),
                 "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
}
// 32 consecutive columns [col0, col0 + 32) of row r (col0 % 32 == 0)
__device__ __forceinline__ void acc_stage_load32(uint32_t stage_smem, uint32_t r, uint32_t col0, uint32_t n,
                                                 uint32_t (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[4 * i]), "=r"(v[4 * i + 1]), "=r"(v[4 * i + 2]), "=r"(v[4 * i + 3])
                 : "r"(stage_smem + acc_stage_offset(r, col0 + 4 * i, n))
                 : "memory");
}

// ----------------------------------------------------------------------------- misc
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
// Byte offset of 16-byte chunk `chunk` (0..7) of row `row` inside a 128B-swizzled tile whose rows are 128 B
// and whose base is 1024-byte aligned (the layout TMA SWIZZLE_128B writes and wgmma SWIZZLE_128B reads).
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128u + ((chunk ^ (row & 7u)) << 4);
}

}  // namespace e2f
