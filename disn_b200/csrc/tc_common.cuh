// sm_90a building blocks for the tensor-core kernels: mbarrier, cluster, register reallocation (setmaxnreg), bulk copy
// (TMA engine), GMMA shared-memory descriptors and warpgroup MMA (wgmma.mma_async, m64n128) wrappers (inline PTX).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- cluster ----------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(cta_rank));
  return r;
}

// ---------------------------------------------------------------- mbarrier ---------------------------
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
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// arrive on the barrier at the same smem offset in CTA `cta_rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta_rank) {
  uint32_t remote = mapa(smem_u32(bar), cta_rank);
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#ifndef DISN_MBAR_TIMEOUT_NS
#define DISN_MBAR_TIMEOUT_NS 4000000000ull   // 4 s: far beyond any legitimate wait in these kernels
#endif
// Bounded wait: a protocol bug traps (reported as a launch failure) instead of hanging the GPU.
// The timer is consulted only every 4096 failed polls: reading %globaltimer costs hundreds of cycles and
// must stay off the common path (try_wait itself suspends the thread until the phase flips or a HW time slice).
// mbar_wait_inline is the whole wait without a call, for a warpgroup that has lowered its register limit
// (setmaxnreg.dec): ptxas fails to allocate a kernel whose reduced-register code calls mbar_wait_slow.
__device__ __forceinline__ void mbar_wait_inline(uint64_t* bar, uint32_t parity) {
  uint64_t t0 = 0;
  for (uint32_t spins = 1;; ++spins) {
    if (mbar_try_wait(bar, parity)) return;
    if ((spins & 0xFFFu) == 0) {
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > DISN_MBAR_TIMEOUT_NS) __trap();
    }
  }
}
static __device__ __noinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity) { mbar_wait_inline(bar, parity); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity);
}

// ---------------------------------------------------------------- register reallocation ---------------
// Change the calling warpgroup's per-thread register limit to N (24..256, a multiple of 8).  Every warp of the
// warpgroup must execute the same instruction.  `dec` returns registers to the CTA's pool; `inc` blocks until the pool
// can grant them, so a kernel that splits roles decreases in one warpgroup what it increases in the others.
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() {
  static_assert(N >= 24 && N <= 256 && N % 8 == 0, "setmaxnreg: 24..256 in steps of 8");
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() {
  static_assert(N >= 24 && N <= 256 && N % 8 == 0, "setmaxnreg: 24..256 in steps of 8");
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------- proxies / fences -------------------
// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- bulk copy (TMA engine, 1-D) --------
// global -> this CTA's shared memory, completion counted in bytes on a local mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// L1 prefetch of the 128-byte line holding `p` (generic address of global memory); a pure hint
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.L1 [%0];" ::"l"(p)); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- operand tiles ----------------------
// K-major SWIZZLE_128B tile of 2-byte elements: rows of 64 elements (128 B), 8-row groups 1024 B apart, tile base
// 1024-B aligned.  Byte offset of 16-byte chunk `chunk` (0..7) of row `row`:
__host__ __device__ constexpr uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return (row >> 3) * 1024u + (row & 7u) * 128u + ((chunk ^ (row & 7u)) << 4);
}
// K-major SWIZZLE_64B tile of 1-byte elements: rows of 64 B, 8-row groups 512 B apart
__host__ __device__ constexpr uint32_t sw64_offset(uint32_t row, uint32_t chunk) {
  return (row >> 3) * 512u + (row & 7u) * 64u + ((chunk ^ ((row >> 1) & 3u)) << 4);
}

// GMMA shared-memory matrix descriptor (sm_90): start address >> 4 in [0,14), leading byte offset >> 4 in [16,30)
// (unused for swizzled K-major tiles, 1), stride byte offset >> 4 in [32,46) (one 8-row group), swizzle mode in
// [62,64) (1 = 128 B, 2 = 64 B).  Moving along K inside the swizzle atom adds bytes >> 4 to the start address.
constexpr uint32_t kDescHiSw128 = 64u | (1u << 30);
constexpr uint32_t kDescHiSw64 = 32u | (2u << 30);
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr) {
  return ((uint64_t)kDescHiSw128 << 32) | (uint64_t)(((smem_addr >> 4) & 0x3FFFu) | (1u << 16));
}
__device__ __forceinline__ uint64_t desc_sw64(uint32_t smem_addr) {
  return ((uint64_t)kDescHiSw64 << 32) | (uint64_t)(((smem_addr >> 4) & 0x3FFFu) | (1u << 16));
}

// ---------------------------------------------------------------- warpgroup MMA ----------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait points
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// operand kinds of wgmma_m64n128: 2-byte kinds take K = 16 per instruction, e5m2 takes K = 32
enum { KIND_BF16 = 0, KIND_F16 = 1, KIND_E5M2 = 2 };

#define DISN_WGMMA_D64                                                                                                \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "   \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define DISN_WGMMA_OPS64                                                                                             \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),       \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),         \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),        \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),        \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),        \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),        \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),        \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] (+)= A[64 x K] * B[128 x K]^T, both operands K-major in shared memory, fp32 accumulators in registers.
// Fragment of thread t of the warpgroup (warp w = t/32, lane l): d[4j + e] = D[16w + l/4 + 8(e/2)][8j + 2(l%4) + e%2].
template <int kKind>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (kKind == KIND_BF16) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " DISN_WGMMA_D64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : DISN_WGMMA_OPS64
                 : "l"(da), "l"(db), "r"(accumulate));
  } else if constexpr (kKind == KIND_F16) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " DISN_WGMMA_D64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : DISN_WGMMA_OPS64
                 : "l"(da), "l"(db), "r"(accumulate));
  } else {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k32.f32.e5m2.e5m2 " DISN_WGMMA_D64 ", %64, %65, p, 1, 1;\n\t}"
                 : DISN_WGMMA_OPS64
                 : "l"(da), "l"(db), "r"(accumulate));
  }
}

// Low word of a descriptor (start address >> 4 and the leading byte offset); the high word is a constant per swizzle
// mode.  Moving the start address by `off` bytes (a multiple of 16, staying inside shared memory, whose addresses
// fit the 14-bit field) adds off >> 4 to it, so the descriptors of one operand tile are one add apart.
__device__ __forceinline__ uint32_t desc_lo(uint32_t smem_addr) { return ((smem_addr >> 4) & 0x3FFFu) | (1u << 16); }

// wgmma_m64n128 with both operands given by descriptor low words: SW128 (KIND_BF16, KIND_F16) or SW64 (KIND_E5M2)
// tiles.  The 64-bit descriptors are formed inside the asm from the constant high word, so the compiler does no
// 64-bit descriptor arithmetic per instruction.
template <int kKind>
__device__ __forceinline__ void wgmma_m64n128_lo(float (&d)[64], uint32_t da, uint32_t db, uint32_t accumulate) {
  constexpr uint32_t hi = kKind == KIND_E5M2 ? kDescHiSw64 : kDescHiSw128;
#define DISN_WGMMA_LO_PRE                                                                                        \
  "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                         \
  "mov.b64 da, {%64, %67};\n\tmov.b64 db, {%65, %67};\n\t"
  if constexpr (kKind == KIND_BF16) {
    asm volatile(DISN_WGMMA_LO_PRE
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " DISN_WGMMA_D64 ", da, db, p, 1, 1, 0, 0;\n\t}"
                 : DISN_WGMMA_OPS64
                 : "r"(da), "r"(db), "r"(accumulate), "r"(hi));
  } else if constexpr (kKind == KIND_F16) {
    asm volatile(DISN_WGMMA_LO_PRE
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " DISN_WGMMA_D64 ", da, db, p, 1, 1, 0, 0;\n\t}"
                 : DISN_WGMMA_OPS64
                 : "r"(da), "r"(db), "r"(accumulate), "r"(hi));
  } else {
    asm volatile(DISN_WGMMA_LO_PRE
                 "wgmma.mma_async.sync.aligned.m64n128k32.f32.e5m2.e5m2 " DISN_WGMMA_D64 ", da, db, p, 1, 1;\n\t}"
                 : DISN_WGMMA_OPS64
                 : "r"(da), "r"(db), "r"(accumulate), "r"(hi));
  }
#undef DISN_WGMMA_LO_PRE
}

#undef DISN_WGMMA_D64
#undef DISN_WGMMA_OPS64

// split fp32 pair into packed bf16 hi and packed bf16 lo (x ~= hi + lo, |x - hi - lo| <= 2^-17 |x|)
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  float ra = a - __low2float(h), rb = b - __high2float(h);
  __nv_bfloat162 l = __floats2bfloat162_rn(ra, rb);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

}  // namespace tc
