// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma, cluster addressing. Nothing here is library code; every wrapper is one PTX instruction (or a bounded
// spin around one) so that the kernels in siglip_kernels.cu read as the hardware sequence they are.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace siglip {

// ---------------------------------------------------------------------------------------------
// Debug record: written to host-mapped pinned memory just before a __trap() so the host can say
// WHICH wait timed out even though the context is dead afterwards.
// ---------------------------------------------------------------------------------------------
struct DebugRecord {
  unsigned int code;    // 0 = ok; else site id of the timed-out wait
  unsigned int block;
  unsigned int thread;
  unsigned int aux0;
  unsigned int aux1;
  unsigned int aux2;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// shared::cta address -> shared::cluster address of the same offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}

__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Arrive on a barrier that lives in another CTA of the cluster (address from mapa_shared).
// Hand-back of a shared-memory stage that was read only by wgmma (async proxy, complete after wgmma.wait_group): the
// arrive has to follow that wait in program order and publishes no memory writes, so it needs no release fence — a
// release at cluster scope costs two full fences (MEMBAR.ALL.CTA + MEMBAR.ALL.GPU) per warp and k block.
__device__ __forceinline__ void mbar_arrive_cluster_relaxed(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}

#ifndef SIGLIP_WAIT_TIMEOUT_NS
#define SIGLIP_WAIT_TIMEOUT_NS 4000000000ull  // 4 s: any legitimate in-kernel wait is < 100 ms
#endif

__device__ __forceinline__ long long clock_cycles() {
  long long c;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(c));
  return c;
}

// Bounded wait: a protocol bug must not hang the GPU. On timeout the site id is published to the
// host-mapped debug record and the kernel traps (the launch then fails loudly on the host).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, DebugRecord* dbg, uint32_t site,
                                          uint32_t aux0 = 0, uint32_t aux1 = 0, uint32_t sleep_ns = 0,
                                          long long* waited = nullptr) {
  if (mbar_try_wait(bar, parity)) return;
  const long long c0 = waited ? clock_cycles() : 0;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (sleep_ns) __nanosleep(sleep_ns);  // long waits (epilogue warps during a K loop): do not burn issue slots
    if ((++spins & 0x3ffu) == 0) {
      uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > SIGLIP_WAIT_TIMEOUT_NS) {
        if (dbg != nullptr) {
          dbg->block = blockIdx.x;
          dbg->thread = threadIdx.x;
          dbg->aux0 = aux0;
          dbg->aux1 = aux1;
          dbg->aux2 = parity;
          dbg->code = site;
          __threadfence_system();
        }
        __trap();
      }
    }
  }
  if (waited) *waited += clock_cycles() - c0;
}

// The same wait for a warp whose 32 lanes all poll (warp-uniform loops of the TMA producer / MMA issuer): the warp
// votes on the outcome, so the control flow around the wait is uniform for the compiler as well and the loop's
// counters, barrier addresses and descriptors can stay in uniform registers.
__device__ __forceinline__ void mbar_wait_warp(uint32_t bar, uint32_t parity, DebugRecord* dbg, uint32_t site,
                                               uint32_t aux0 = 0, uint32_t aux1 = 0, long long* waited = nullptr) {
  if (__all_sync(0xffffffffu, mbar_try_wait(bar, parity))) return;
  const long long c0 = waited ? clock_cycles() : 0;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (!__all_sync(0xffffffffu, mbar_try_wait(bar, parity))) {
    if ((++spins & 0x3ffu) == 0) {
      uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > SIGLIP_WAIT_TIMEOUT_NS) {
        if (dbg != nullptr) {
          dbg->block = blockIdx.x;
          dbg->thread = threadIdx.x;
          dbg->aux0 = aux0;
          dbg->aux1 = aux1;
          dbg->aux2 = parity;
          dbg->code = site;
          __threadfence_system();
        }
        __trap();
      }
    }
  }
  if (waited) *waited += clock_cycles() - c0;
}

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// 2-D tiled load global -> shared, completion (bytes) signalled on `bar`.
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// L2 eviction-priority policies for streamed vs re-used operands (createpolicy; whole line range, fraction 1.0).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// tma_load_2d with an L2 cache policy for the lines it touches.
__device__ __forceinline__ void tma_load_2d_hint(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1,
                                                 uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// Same load, delivered to the same shared-memory offset of every CTA in `cta_mask` of the cluster; each
// destination CTA's barrier at offset `bar` receives the complete_tx. One L2 read feeds all destinations.
__device__ __forceinline__ void tma_load_2d_mcast(const CUtensorMap* m, uint32_t bar, uint32_t dst, int c0, int c1,
                                                  uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5}], [%2], %3;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "h"(cta_mask), "r"(c0), "r"(c1)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): D[64 x 128, fp32 registers] (+)= A[smem desc] * B[smem desc]
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kN>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kN) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs.
__device__ __forceinline__ void acc_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

#define SIGLIP_WGMMA_ACC64                                                                                         \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "    \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define SIGLIP_WGMMA_OUT64(d)                                                                                      \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),        \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),         \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),        \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),        \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),        \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),        \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),        \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// Operand type of the MMA: 0 bf16 x bf16, 1 fp16 x fp16 (K = 16 per instruction), 2 e4m3 x e4m3 (K = 32, K-major only).
// kTA / kTB: 1 = the operand is MN-major in shared memory (transposed), 0 = K-major.
template <int kType, int kTA, int kTB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (kType == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " SIGLIP_WGMMA_ACC64 ", %64, %65, p, 1, 1, %67, %68;\n\t}"
        : SIGLIP_WGMMA_OUT64(d)
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTA), "n"(kTB));
  } else if constexpr (kType == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " SIGLIP_WGMMA_ACC64 ", %64, %65, p, 1, 1, %67, %68;\n\t}"
        : SIGLIP_WGMMA_OUT64(d)
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTA), "n"(kTB));
  } else {
    static_assert(kType != 2 || (kTA == 0 && kTB == 0), "8-bit wgmma operands are K-major");
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 " SIGLIP_WGMMA_ACC64 ", %64, %65, p, 1, 1;\n\t}"
        : SIGLIP_WGMMA_OUT64(d)
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
  }
}

// D[64 x 256] (+)= A * B: the gradient kernel's 256-column tiles, 16-bit operands only (the same transpose bits).
#define SIGLIP_WGMMA_ACC128                                                                                         \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "    \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, "    \
  "%68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, "    \
  "%90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, "    \
  "%110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
template <int kType, int kTA, int kTB>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(kType == 0 || kType == 1, "m64n256: bf16 or fp16 operands");
  float* h = d + 64;   // second half of the fragment: columns 128 .. 255
  if constexpr (kType == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " SIGLIP_WGMMA_ACC128
        ", %128, %129, p, 1, 1, %131, %132;\n\t}"
        : SIGLIP_WGMMA_OUT64(d), SIGLIP_WGMMA_OUT64(h)
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTA), "n"(kTB));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " SIGLIP_WGMMA_ACC128
        ", %128, %129, p, 1, 1, %131, %132;\n\t}"
        : SIGLIP_WGMMA_OUT64(d), SIGLIP_WGMMA_OUT64(h)
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTA), "n"(kTB));
  }
}
#undef SIGLIP_WGMMA_ACC128
#undef SIGLIP_WGMMA_ACC64
#undef SIGLIP_WGMMA_OUT64


// ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of wgmma (PTX ISA "Matrix Descriptor Format", sm_90), 128-byte swizzle:
//   [0,14)  start address >> 4      [16,30) leading byte offset >> 4
//   [32,46) stride byte offset >> 4 [62,64) swizzle mode (1 = 128B)
// K-major: 8-row groups SBO = 1024 B apart (LBO unused). MN-major: 64-element MN blocks LBO apart, 8-k groups SBO apart.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ---------------------------------------------------------------------------------------------
// MUFU approximations (each one SFU instruction)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace siglip
