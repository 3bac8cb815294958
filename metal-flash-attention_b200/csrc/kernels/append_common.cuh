// Device helpers of the paged K/V appends (paged_append.cu, rotary_append.cu): vector units of a run of elements, the
// E4M3 quantization of a source value, and the slot of a new token.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_params.h"

namespace mfa {
namespace {

constexpr uint32_t kAppendTokens = 16;       // tokens per CTA
constexpr uint32_t kAppendThreads = 256;     // per CTA, at most
constexpr uint32_t kSkip = 0xffffffffu;      // pool_row of a token that is not written
constexpr float kE4m3Max = 448.0f;

template <int kPrec>
struct Element {
  using T = uint16_t;
};
template <>
struct Element<FP32> {
  using T = float;
};

// kWidth consecutive elements of one run.  kWidth == 1: one element (the scalar instantiation, any alignment); else
// kWidth * element bytes is 16 or 32, read as 16-byte vectors
template <int kPrec, int kWidth>
struct Unit {
  static constexpr int kBytes = kWidth * (kPrec == FP32 ? 4 : 2);
  static constexpr int kVectors = kBytes >= 16 ? kBytes / 16 : 1;
  uint4 v[kVectors];

  __device__ __forceinline__ void load(const typename Element<kPrec>::T *__restrict__ p) {
    if constexpr (kWidth == 1 && kPrec == FP32) {
      v[0].x = __float_as_uint(__ldg(p));
    } else if constexpr (kWidth == 1) {
      v[0].x = __ldg(p);
    } else {
#pragma unroll
      for (int i = 0; i < kVectors; ++i) v[i] = __ldg(reinterpret_cast<const uint4 *>(p) + i);
    }
  }
  __device__ __forceinline__ void store(typename Element<kPrec>::T *__restrict__ p) const {
    if constexpr (kWidth == 1 && kPrec == FP32) {
      *p = __uint_as_float(v[0].x);
    } else if constexpr (kWidth == 1) {
      *p = static_cast<uint16_t>(v[0].x);
    } else {
#pragma unroll
      for (int i = 0; i < kVectors; ++i) reinterpret_cast<uint4 *>(p)[i] = v[i];
    }
  }
  // element j converted exactly to FP32
  __device__ __forceinline__ float at(int j) const {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(v);
    if constexpr (kPrec == FP32) {
      return __uint_as_float(w[j]);
    } else {
      const uint32_t bits = (w[j / 2] >> (16 * (j % 2))) & 0xffffu;
      if constexpr (kPrec == BF16) {
        return __uint_as_float(bits << 16);
      } else {
        float f;
        asm("{\n"
            ".reg .b16 h;\n"
            "cvt.u16.u32 h, %1;\n"
            "cvt.f32.f16 %0, h;\n"
            "}\n"
            : "=f"(f)
            : "r"(bits));
        return f;
      }
    }
  }
};
// x / scale rounded to nearest (IEEE division, as torch divides), saturated to the largest finite E4M3 value; NaN stays
// NaN.  The explicit clamp makes +-inf +-448 whatever the conversion does with infinities; finite quotients beyond 448
// round to 448 in either case
__device__ __forceinline__ float e4m3_quotient(float x, float scale) {
  const float q = __fdiv_rn(x, scale);
  return fabsf(q) > kE4m3Max ? copysignf(kE4m3Max, q) : q;
}
// two quotients -> two E4M3 bytes, `lo` in the low byte
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// The unit's kWidth elements quantized with `scale` and stored as kWidth bytes (8 or 16 bytes in one store, or 1)
template <int kPrec, int kWidth>
__device__ __forceinline__ void store_e4m3(const Unit<kPrec, kWidth> &u, float scale, uint8_t *__restrict__ p) {
  if constexpr (kWidth == 1) {
    *p = static_cast<uint8_t>(e4m3x2(e4m3_quotient(u.at(0), scale), 0.0f) & 0xffu);
  } else {
    static_assert(kWidth == 8 || kWidth == 16, "8 or 16 bytes per store");
    uint32_t w[kWidth / 4];
#pragma unroll
    for (int i = 0; i < kWidth / 4; ++i)
      w[i] = e4m3x2(e4m3_quotient(u.at(4 * i), scale), e4m3_quotient(u.at(4 * i + 1), scale)) |
             (e4m3x2(e4m3_quotient(u.at(4 * i + 2), scale), e4m3_quotient(u.at(4 * i + 3), scale)) << 16);
    if constexpr (kWidth == 16)
      *reinterpret_cast<uint4 *>(p) = make_uint4(w[0], w[1], w[2], w[3]);
    else
      *reinterpret_cast<uint2 *>(p) = make_uint2(w[0], w[1]);
  }
}

// The pool row of new token i of sequence s (span: the sequence's paged_span): key p = Cs - Rs + i, row
// page_table[s][p / P] * P + p % P.  kSkip for i >= Rs or p < 0, and for a page id outside [0, pages): a write is
// skipped, never clamped, so a malformed table cannot redirect it into another sequence's page.  *position receives p
// when p >= 0 and is left as it is otherwise.  (paged_kv_append spells the same rule out inline: through this helper
// ptxas orders one comparison differently, and its SASS is kept byte for byte.)
__device__ __forceinline__ uint32_t token_slot(const PagedKV &pk, const SequenceSpan &span, uint32_t s, uint32_t i,
                                               uint32_t *position) {
  uint32_t row = kSkip;
  if (i < span.R) {
    const int64_t p = static_cast<int64_t>(span.C) - static_cast<int64_t>(span.R) + i;
    if (p >= 0) {  // (p < Cs <= max_keys = page_stride * P: the entry is inside the sequence's page_table row)
      const uint32_t key = static_cast<uint32_t>(p);
      *position = key;
      const int page = __ldg(pk.page_table + static_cast<uint64_t>(s) * pk.page_stride + (key >> pk.page_shift));
      if (page >= 0 && static_cast<uint32_t>(page) < pk.pages)
        row = (static_cast<uint32_t>(page) << pk.page_shift) | (key & ((1u << pk.page_shift) - 1));
    }
  }
  return row;
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace
}  // namespace mfa
