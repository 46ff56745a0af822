// sm_90a PTX building blocks shared by the jenga_b200 kernels: mbarrier, TMA
// (cp.async.bulk.tensor), warpgroup MMA (wgmma.mma_async, fence / commit / wait) and its
// shared-memory matrix descriptor.  Everything here is inline PTX; there is no CUTLASS
// dependency.  The descriptor layout follows the PTX ISA "Matrix Descriptor Format" table of the
// asynchronous warpgroup-level matrix instructions.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace jenga {

// ---------------------------------------------------------------------------------------------
// Error codes written to the device-side error flag by watchdogs (see mbar_wait).
// ---------------------------------------------------------------------------------------------
enum : int {
  JENGA_DEV_OK = 0,
  JENGA_DEV_WATCHDOG = 0x7001,  // an mbarrier wait exceeded the watchdog budget
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must never hang the GPU box.  After ~2^31 cycles (about a
// second) the waiter records JENGA_DEV_WATCHDOG in *err_flag and traps, which surfaces on the
// host as a launch failure instead of a hang.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* err_flag) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  for (;;) {
    // tight inner loop: try_wait suspends the thread in hardware until the phase flips or a
    // time limit passes, so 256 probes are cheap in issue slots
#pragma unroll 1
    for (int i = 0; i < 256; ++i)
      if (mbar_try_wait(bar, parity)) return;
    if ((clock64() - t0) > (1ll << 31)) {
      if (err_flag) atomicExch(err_flag, JENGA_DEV_WATCHDOG);
      __threadfence_system();
      __trap();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Proxy fence: generic-proxy shared-memory writes -> visible to TMA / wgmma (async proxy)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// TMA: 4-D tiled load global -> shared, completion on an mbarrier (transaction bytes)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a).  All four warps of a warpgroup execute these together.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// keeps the compiler from moving accumulator accesses across an in-flight wgmma
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// Shared-memory matrix descriptor (64-bit):
//   [ 0,14) start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4   [49,52) base offset (0: atoms are 1024-B aligned)
//   [62,64) layout (1 = SWIZZLE_128B)
// K-major SW128: 8-row groups are SBO apart, LBO unused.  MN-major SW128: 64-element MN chunks are
// LBO apart, 8-row K groups SBO apart.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= 1ull << 62;
  return d;
}

// the 64 fp32 accumulator registers of an m64n128 wgmma: operands %0..%63
#define JENGA_WGMMA_D64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define JENGA_WGMMA_OUT64 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define JENGA_WGMMA_SS(TY)                                                                              \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                        \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " " JENGA_WGMMA_D64             \
               ", %64, %65, p, 1, 1, 0, 0;\n\t}\n"                                                     \
               : JENGA_WGMMA_OUT64 : "l"(a_desc), "l"(b_desc), "r"(scale_d))
#define JENGA_WGMMA_RS(SHAPE, TY, TAIL)                                                                 \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"                                        \
               "wgmma.mma_async.sync.aligned." SHAPE ".f32." TY "." TY " " JENGA_WGMMA_D64              \
               ", {%64, %65, %66, %67}, %68, p, 1, 1" TAIL ";\n\t}\n"                                  \
               : JENGA_WGMMA_OUT64 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d))

// D[64x128 f32, registers] (+)= A[smem, K-major] * B[smem, K-major], K = 16 (16-bit operands)
template <bool kBF16>
__device__ __forceinline__ void wgmma_128_ss(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (kBF16) JENGA_WGMMA_SS("bf16");
  else JENGA_WGMMA_SS("f16");
}
// D[64x128 f32] (+)= A[registers] * B[smem, MN-major], K = 16 (16-bit operands)
template <bool kBF16>
__device__ __forceinline__ void wgmma_128_rs_bmn(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc,
                                                 uint32_t scale_d) {
  if constexpr (kBF16) JENGA_WGMMA_RS("m64n128k16", "bf16", ", 1");
  else JENGA_WGMMA_RS("m64n128k16", "f16", ", 1");
}
// D[64x128 f32] (+)= A[registers] * B[smem, K-major], K = 32, e4m3 x e4m3 (8-bit operands are K-major only)
__device__ __forceinline__ void wgmma_128_rs_e4m3(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc,
                                                  uint32_t scale_d) {
  JENGA_WGMMA_RS("m64n128k32", "e4m3", "");
}
// four fp32 -> packed e4m3x4 (byte i = value i), round-to-nearest, saturating
__device__ __forceinline__ uint32_t pack4_e4m3(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
}

// sub-CTA barrier among `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------------------------------------
// Small numeric helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// {hi, lo} fp32 -> packed 16-bit pair, round-to-nearest-even (lo lands in bits [0,16)).
template <bool kBF16>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  uint32_t r;
  if constexpr (kBF16) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  } else {
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  }
  return r;
}
template <bool kBF16>
__device__ __forceinline__ float2 unpack2(uint32_t v) {
  float2 f;
  if constexpr (kBF16) {
    f.x = __uint_as_float(v << 16);
    f.y = __uint_as_float(v & 0xffff0000u);
  } else {
    asm("{\n\t.reg .b16 lo, hi;\n\tmov.b32 {lo, hi}, %2;\n\t"
        "cvt.f32.f16 %0, lo;\n\tcvt.f32.f16 %1, hi;\n\t}\n"
        : "=f"(f.x), "=f"(f.y)
        : "r"(v));
  }
  return f;
}

}  // namespace jenga
