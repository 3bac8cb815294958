// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and the wgmma shared-memory descriptor
// (wgmma.cuh has the MMA instructions).  Hand-written for this repository; bit layouts follow the PTX ISA "wgmma"
// chapter (the same layouts CUTLASS documents in cute/arch/mma_sm90_desc.hpp).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mfa {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ uint32_t lane_id() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(r));
  return r;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

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

// ---------------------------------------------------------------- streaming global loads -----
// Read-once data (O and dO rows for D = rowsum(dO * O)): no L1 line is allocated for the miss (the kernels leave
// little L1 beside their shared memory).
__device__ __forceinline__ float4 ldg_stream_f32x4(const float *p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ uint2 ldg_stream_u32x2(const void *p) {
  uint2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
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

// 3-D tiled store shared -> global (bulk async-group completion).  The issuing THREAD owns the group: the same thread
// commits and later waits.  Generic-proxy writes to the source tile need fence.proxy.async before the store is issued.
__device__ __forceinline__ void tma_store_3d(const void *map, uint32_t smem_src, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed group of this thread has finished READING shared memory (the source tile may be rewritten)
__device__ __forceinline__ void tma_store_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... has completed (the global writes are done)
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// 1-D bulk copy global -> shared (no tensor map): `bytes` a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
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

// ---------------------------------------------------------------- shared memory, explicit state space ----
// Pointers derived from the manually aligned dynamic shared-memory base are generic to the compiler (LD.E / ST.E in
// SASS); the staging tiles of the epilogues go through these instead so that they compile to LDS / STS.
__device__ __forceinline__ void sts_f32x4(uint32_t addr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds_f32x4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
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

// the two 16-bit halves of a packed register, widened back to FP32 (exact)
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t w) {
  return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u));
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t w) {
  float2 r;
  asm("{\n"
      ".reg .b16 lo, hi;\n"
      "mov.b32 {lo, hi}, %2;\n"
      "cvt.f32.f16 %0, lo;\n"
      "cvt.f32.f16 %1, hi;\n"
      "}\n"
      : "=f"(r.x), "=f"(r.y)
      : "r"(w));
  return r;
}

// ---------------------------------------------------------------- register reallocation ------
template <uint32_t RegCount>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(RegCount));
}
template <uint32_t RegCount>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(RegCount));
}

}  // namespace ptx
}  // namespace mfa
