// Thin inline-PTX wrappers for sm_90a: mbarrier, bulk async copy (TMA), wgmma.
// Everything here is hand-written for Hopper; there is no fallback path.
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace dmd {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(1000000u)  // suspend-time hint (ns): sleep instead of busy-polling
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a launch error (trap), never as a hung GPU.  A failed try_wait suspends for
// an implementation-defined time up to the 1 ms hint (observed: microseconds), so 2^20 failures is seconds to minutes on
// one phase -- orders of magnitude beyond the longest legitimate wait of any kernel here.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 20)) asm volatile("trap;");
  }
}

// ---------------------------------------------------------------- proxies / fences
// generic-proxy smem writes (st.shared) -> visible to the async proxy (wgmma operand reads, TMA)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- bulk async copy (TMA 1-D), global -> smem
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---------------------------------------------------------------- wgmma shared-memory matrix descriptors
// SWIZZLE_NONE ("interleave") canonical layouts, 16-byte units:
//   K-major : core matrix = 8 MN-rows x 16 B (8 k-elements), contiguous 128 B; LBO = stride of the 8-element K chunks,
//             SBO = stride of the 8-row MN groups
//   MN-major: core matrix = 8 k-rows x 16 B (8 MN-elements), contiguous 128 B; LBO = stride of the 8-row K groups,
//             SBO = stride of the 8-element MN groups
// bits [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout (0 = no swizzle).  The start address only has to be
// 16-byte aligned, so a descriptor can address a window shifted by any whole number of 16-byte rows (the conv taps).
__host__ __device__ __forceinline__ uint64_t gmma_desc_hi(uint32_t sbo_bytes) {
  return (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
}
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return gmma_desc_hi(sbo_bytes) | (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16);
}

// ---------------------------------------------------------------- wgmma (one warpgroup, fp16 x fp16 -> fp32 registers)
// D[64 x N] (+)= A[64 x 16] * B[16 x N], both operands in shared memory.  Fragment of D held by thread t of the warpgroup
// (warp w = t / 32, lane l):  d[4j + 2s + e] = D[16w + l/4 + 8s][8j + 2(l%4) + e].  kTransA / kTransB: 0 = K-major,
// 1 = MN-major operand.
template <int N>
struct Wgmma;
template <>
struct Wgmma<16> {
  template <int kTransA, int kTransB>
  __device__ __forceinline__ static void mma(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};
template <>
struct Wgmma<32> {
  template <int kTransA, int kTransB>
  __device__ __forceinline__ static void mma(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};
template <>
struct Wgmma<64> {
  template <int kTransA, int kTransB>
  __device__ __forceinline__ static void mma(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};
template <>
struct Wgmma<128> {
  template <int kTransA, int kTransB>
  __device__ __forceinline__ static void mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Orders the compiler's accesses of accumulator registers against the asynchronous wgmma (no instruction is emitted).
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// launch_dependents: the next kernel in the stream (launched with the programmatic-serialization attribute) may start
// its prologue now.  wait: block until the previous kernel has completed and its memory is visible.
// elect.sync: one lane of a CONVERGED warp (deterministic for a given mask).  Code under `if (elect_one_sync())` keeps
// warp-uniform values in uniform registers, which is what cp.async.bulk wants.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- kernel trace (diagnostics)
// One thread stores the GPU's nanosecond timer once the kernel's dependencies are satisfied: consecutive stamps of a stream of
// kernels give the in-graph duration of each (scripts/ktrace.py).  A null pointer (the production setting) costs one test.
__device__ __forceinline__ void ktrace_stamp(long long* slot) {
  if (slot != nullptr) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    *slot = (long long)t;
  }
}

// ---------------------------------------------------------------- small math
// SiLU with the bare SFU approximations (5 instructions): v * rcp(1 + 2^(-v*log2 e)).  ex2/rcp.approx.ftz carry ~2 ulp;
// 1 + e >= 1 so rcp needs no range fix-up (e = +inf -> 0), unlike __fdividef / __expf which add ~4 instructions each.
__device__ __forceinline__ float silu_f(float v) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return v * r;
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace dmd
