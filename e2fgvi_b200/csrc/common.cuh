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
__device__ __forceinline__ void tma_load_4d(uint32_t smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
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

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, A and B K-major in shared memory, issued by a whole warpgroup as ONE
// m64nNk16 instruction.  Accumulator fragment of thread t (warp w = (t / 32) % 4, lane l): d[4j + {0,1}] = row 16w + l/4,
// columns 8j + 2(l%4) + {0,1}; d[4j + {2,3}] = the same columns of row 16w + l/4 + 8.  acc = 0 overwrites D.
// Every instruction reads its whole 2 KB A tile from shared memory, so one full-width instruction instead of several
// 64-column ones cuts the A traffic: m64n64k16 alone needs 128 B/clk of shared memory at the tensor pipe's rate, all an
// SM has; m64n128k16 needs 96 and m64n256k16 80.  B rows are contiguous 128-byte K rows (8-row groups 1024 B apart).
//
// Operand lists: E2F_WR<c> names accumulator registers 8c .. 8c + 7 in the PTX string, E2F_WD<n>(i) binds d[i .. i + n).
#define E2F_WR0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define E2F_WR1 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define E2F_WR2 ", %16, %17, %18, %19, %20, %21, %22, %23"
#define E2F_WR3 ", %24, %25, %26, %27, %28, %29, %30, %31"
#define E2F_WR4 ", %32, %33, %34, %35, %36, %37, %38, %39"
#define E2F_WR5 ", %40, %41, %42, %43, %44, %45, %46, %47"
#define E2F_WR6 ", %48, %49, %50, %51, %52, %53, %54, %55"
#define E2F_WR7 ", %56, %57, %58, %59, %60, %61, %62, %63"
#define E2F_WR8 ", %64, %65, %66, %67, %68, %69, %70, %71"
#define E2F_WR9 ", %72, %73, %74, %75, %76, %77, %78, %79"
#define E2F_WR10 ", %80, %81, %82, %83, %84, %85, %86, %87"
#define E2F_WR11 ", %88, %89, %90, %91, %92, %93, %94, %95"
#define E2F_WR12 ", %96, %97, %98, %99, %100, %101, %102, %103"
#define E2F_WR13 ", %104, %105, %106, %107, %108, %109, %110, %111"
#define E2F_WR14 ", %112, %113, %114, %115, %116, %117, %118, %119"
#define E2F_WR15 ", %120, %121, %122, %123, %124, %125, %126, %127"
#define E2F_WD8(i) "+f"(d[(i)]), "+f"(d[(i) + 1]), "+f"(d[(i) + 2]), "+f"(d[(i) + 3]), \
                   "+f"(d[(i) + 4]), "+f"(d[(i) + 5]), "+f"(d[(i) + 6]), "+f"(d[(i) + 7])
#define E2F_WD16(i) E2F_WD8(i), E2F_WD8((i) + 8)
#define E2F_WD32(i) E2F_WD16(i), E2F_WD16((i) + 16)
#define E2F_WD64(i) E2F_WD32(i), E2F_WD32((i) + 32)

// one specialisation per (N, f16) the kernels use; any other width fails to compile
template <int N, bool F16>
struct WgmmaSS;
// IA / IB / IP: operand numbers of the A descriptor, the B descriptor and the accumulate flag (N/2, N/2 + 1, N/2 + 2)
#define E2F_WGMMA_SS(N, F16, TY, REGS, IA, IB, IP, ...)                                                              \
  template <>                                                                                                       \
  struct WgmmaSS<N, F16> {                                                                                          \
    static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {            \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" IP ", 0;\n"                                                 \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" REGS "}, %" IA ", %" IB         \
                   ", p, 1, 1, 0, 0;\n}\n"                                                                          \
                   : __VA_ARGS__                                                                                    \
                   : "l"(adesc), "l"(bdesc), "r"(acc));                                                             \
    }                                                                                                               \
  };
E2F_WGMMA_SS(32, false, "bf16", E2F_WR0 E2F_WR1, "16", "17", "18", E2F_WD16(0))
E2F_WGMMA_SS(48, false, "bf16", E2F_WR0 E2F_WR1 E2F_WR2, "24", "25", "26", E2F_WD16(0), E2F_WD8(16))
E2F_WGMMA_SS(64, false, "bf16", E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3, "32", "33", "34", E2F_WD32(0))
E2F_WGMMA_SS(96, false, "bf16", E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5, "48", "49", "50", E2F_WD32(0),
             E2F_WD16(32))
E2F_WGMMA_SS(112, false, "bf16", E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5 E2F_WR6, "56", "57", "58",
             E2F_WD32(0), E2F_WD16(32), E2F_WD8(48))
E2F_WGMMA_SS(128, false, "bf16", E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5 E2F_WR6 E2F_WR7, "64", "65", "66",
             E2F_WD64(0))
E2F_WGMMA_SS(224, false, "bf16",
             E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5 E2F_WR6 E2F_WR7 E2F_WR8 E2F_WR9 E2F_WR10 E2F_WR11 E2F_WR12
                 E2F_WR13,
             "112", "113", "114", E2F_WD64(0), E2F_WD32(64), E2F_WD16(96))
E2F_WGMMA_SS(256, false, "bf16",
             E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5 E2F_WR6 E2F_WR7 E2F_WR8 E2F_WR9 E2F_WR10 E2F_WR11 E2F_WR12
                 E2F_WR13 E2F_WR14 E2F_WR15,
             "128", "129", "130", E2F_WD64(0), E2F_WD64(64))
E2F_WGMMA_SS(64, true, "f16", E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3, "32", "33", "34", E2F_WD32(0))
E2F_WGMMA_SS(128, true, "f16", E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 E2F_WR4 E2F_WR5 E2F_WR6 E2F_WR7, "64", "65", "66",
             E2F_WD64(0))

template <int N, bool F16>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  WgmmaSS<N, F16>::run(d, adesc, bdesc, acc);
}
// register-A variant (A fragment in registers, B transposed = MN-major in shared memory)
__device__ __forceinline__ void wgmma_n64_f16_rs_tb(float* d, const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {" E2F_WR0 E2F_WR1 E2F_WR2 E2F_WR3 "}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
      : E2F_WD32(0)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
}

// ----------------------------------------------------------------------------- warp specialisation
// named barriers (id 0 is __syncthreads); `threads` counts every thread that syncs or arrives
__device__ __forceinline__ void named_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// setmaxnreg: a producer warpgroup gives registers back, consumer warpgroups take them (the whole warpgroup executes it)
template <int REGS>
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS>
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }

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
