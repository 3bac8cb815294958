// Pieces shared by the tensor-core kernels (wgmma_attention.cu) and the staging copies (pad_head.cu): statistic loads /
// stores and the BF16 -> FP16 rewrite of dO.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_params.h"
#include "sm90_ptx.cuh"

namespace mfa {
namespace bwd {

using namespace ptx;

__device__ __forceinline__ float load_16bit(const void *p, size_t i, bool bf16) {
  const uint16_t h = reinterpret_cast<const uint16_t *>(p)[i];
  return bf16 ? __uint_as_float(static_cast<uint32_t>(h) << 16) : __half2float(__ushort_as_half(h));
}
// L is FP32 or FP16, D is FP32 or BF16 in memory (AttentionDescriptor+Precisions.swift:81-87)
__device__ __forceinline__ float load_stat(const void *p, size_t i, int prec) {
  if (prec == FP32) return reinterpret_cast<const float *>(p)[i];
  const uint16_t h = reinterpret_cast<const uint16_t *>(p)[i];
  return prec == FP16 ? __half2float(__ushort_as_half(h)) : __uint_as_float(static_cast<uint32_t>(h) << 16);
}
__device__ __forceinline__ void store_stat(void *p, size_t i, int prec, float v) {
  if (prec == FP32) reinterpret_cast<float *>(p)[i] = v;
  else if (prec == FP16) reinterpret_cast<uint16_t *>(p)[i] = __half_as_ushort(__float2half_rn(v));
  else reinterpret_cast<uint16_t *>(p)[i] = static_cast<uint16_t>(__float_as_uint(v) >> 16);  // BF16 store truncates
}

// dO arrives as BF16 while Q, K, V are FP16 (the reference's own low-precision policy,
// AttentionDescriptor+Precisions.swift:13-23); wgmma cannot mix the two element types in one MMA, so dO is
// rewritten as FP16 before any MMA reads it.  BF16 -> FP16 is exact for 2^-14 <= |x| < 65504
// (8 significant bits fit FP16's 11); gradients outside that range would not survive FP16 Q/K/V either.
__device__ __forceinline__ uint32_t bf16x2_to_f16x2(uint32_t w) {
  return pack_f16x2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u));
}
__device__ __forceinline__ uint4 bf16x8_to_f16x8(uint4 v) {
  return make_uint4(bf16x2_to_f16x2(v.x), bf16x2_to_f16x2(v.y), bf16x2_to_f16x2(v.z), bf16x2_to_f16x2(v.w));
}

}  // namespace bwd
}  // namespace mfa
