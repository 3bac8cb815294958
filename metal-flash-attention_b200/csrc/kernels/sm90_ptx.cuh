// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and the wgmma shared-memory descriptor
// (wgmma.cuh has the MMA instructions).  Hand-written for this repository; bit layouts follow the PTX ISA "wgmma"
// chapter (the same layouts CUTLASS documents in cute/arch/mma_sm90_desc.hpp).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mfa {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---------------------------------------------------------------- mbarrier -------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Completes `bytes` of the transaction count the barrier's current phase expects without a copy (loads that a caller
// decided not to issue)
__device__ __forceinline__ void mbar_complete_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.complete_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// Bounded wait: a protocol bug must surface as a trapped kernel (an error the host reports), never
// as a hung GPU.  ~4 s at 2 GHz; the check costs nothing on the fast path.
// A trap from a kernel of this library therefore means a barrier protocol error (a wait whose phase never completes).
// The branch holds no printf: any call in a kernel makes ptxas serialize every wgmma of that kernel (C7510).  To find
// the barrier, block and parity that timed out, add a printf before the __trap locally.
#ifndef MFA_MBAR_TIMEOUT_CYCLES
#define MFA_MBAR_TIMEOUT_CYCLES (8000000000ll)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long start = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity))
    if ((++spins & 0x3ffu) == 0 && clock64() - start > MFA_MBAR_TIMEOUT_CYCLES) __trap();
}

// ---------------------------------------------------------------- TMA ------------------------
__device__ __forceinline__ void prefetch_tensormap(const void *map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 3-D tiled load global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const void *map, uint64_t *bar, int32_t c0, int32_t c1,
                                            int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------- wgmma shared-memory descriptor ----
// 128-byte swizzle (what TMA SWIZZLE_128B writes):
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset = 0 (tiles are 1024-byte aligned)   [62,64) layout type: 1 = SWIZZLE_128B
// K-major operand  (rows = M or N index, 64 16-bit K elements = one 128 B swizzle row):
//   SBO = distance between 8-row groups (1024 B); LBO unused.  A K step of 16 elements advances the start by 32 B.
// MN-major operand (rows = K index, 64 16-bit MN elements per 128 B row):
//   SBO = distance between 8-row (K) groups (1024 B); LBO = distance between 64-element MN blocks.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t desc = 0;
  desc |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  desc |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  desc |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  desc |= static_cast<uint64_t>(1) << 62;
  return desc;
}

// ---------------------------------------------------------------- math helpers ----------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// pack two FP32 into one 32-bit register of 16-bit values: low half = lo, high half = hi
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// four OCP E4M3 bytes (byte 0 lowest) -> two f16x2 registers (byte 0 in the low half of .x); exact, NaN stays NaN
__device__ __forceinline__ uint2 e4m3x4_to_f16x4(uint32_t bytes) {
  uint2 r;
  asm("{\n"
      ".reg .b16 lo, hi;\n"
      "mov.b32 {lo, hi}, %2;\n"
      "cvt.rn.f16x2.e4m3x2 %0, lo;\n"
      "cvt.rn.f16x2.e4m3x2 %1, hi;\n"
      "}\n"
      : "=r"(r.x), "=r"(r.y)
      : "r"(bytes));
  return r;
}
// f16x2 -> bf16x2 through FP32: exact for every value an E4M3 byte holds (at most 4 significant bits, exponent in
// [-9, 8])
__device__ __forceinline__ uint32_t f16x2_to_bf16x2(uint32_t h) {
  float lo, hi;
  asm("{\n"
      ".reg .b16 a, b;\n"
      "mov.b32 {a, b}, %2;\n"
      "cvt.f32.f16 %0, a;\n"
      "cvt.f32.f16 %1, b;\n"
      "}\n"
      : "=f"(lo), "=f"(hi)
      : "r"(h));
  return pack_bf16x2(lo, hi);
}

}  // namespace ptx
}  // namespace mfa
