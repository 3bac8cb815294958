// Paged K/V append (mfa_paged_kv_append): the step's new keys and values, packed by sequence as the paged forward's
// queries are, are written into the page pools through the same table the forward reads.  New token i of sequence s
// (0 <= i < Rs) is key p = Cs - Rs + i, pool row page_table[s][p / P] * P + p % P, every K/V head.  A pool row holds
// one token's Hkv * D elements contiguously, as does the source, so each token is one contiguous run: a copy of 16-byte
// vectors, or a quantization to E4M3 bytes with the K/V head's scale.
//
// One CTA per (kAppendTokens tokens, sequence): its first threads resolve the pool row of each of its tokens once (the
// forward's clamping of the query range and of Cs; a position p < 0 or a page id outside [0, pages) is skipped, never
// clamped, so a malformed table cannot redirect a write into another sequence's page), then the CTA moves the runs.
// threadIdx.x walks the vector units of a run and threadIdx.y the tokens, so each thread reads its unit's scales once.
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

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

// grid (ceil(max_row / kAppendTokens), count), block (units of a run, up to 256 threads; tokens)
template <int kPrec, int kWidth, bool kFp8>
__global__ void __launch_bounds__(kAppendThreads) paged_kv_append(const PagedKV pk, const AppendSource src,
                                                                  void *__restrict__ k_pool,
                                                                  void *__restrict__ v_pool, const Fp8KV fp8) {
  using T = typename Element<kPrec>::T;
  using Out = typename std::conditional<kFp8, uint8_t, T>::type;
  __shared__ uint32_t pool_row[kAppendTokens], token[kAppendTokens];
  const uint32_t s = blockIdx.y;
  if (threadIdx.y == 0 && threadIdx.x < kAppendTokens) {
    const SequenceSpan span = paged_span(pk, s);
    const uint32_t i = blockIdx.x * kAppendTokens + threadIdx.x;
    uint32_t row = kSkip;
    if (i < span.R) {
      const int64_t p = static_cast<int64_t>(span.C) - static_cast<int64_t>(span.R) + i;
      if (p >= 0) {  // (p < Cs <= max_keys = page_stride * P: the entry is inside the sequence's page_table row)
        const uint32_t key = static_cast<uint32_t>(p);
        const int page = __ldg(pk.page_table + static_cast<uint64_t>(s) * pk.page_stride + (key >> pk.page_shift));
        if (page >= 0 && static_cast<uint32_t>(page) < pk.pages)
          row = (static_cast<uint32_t>(page) << pk.page_shift) | (key & ((1u << pk.page_shift) - 1));
      }
    }
    pool_row[threadIdx.x] = row;
    token[threadIdx.x] = span.q0 + i;
  }
  __syncthreads();
  const uint32_t units = src.row_elements / kWidth;
  for (uint32_t u = threadIdx.x; u < units; u += blockDim.x) {
    float k_scale = 1.0f, v_scale = 1.0f;
    if constexpr (kFp8) {  // (a unit never straddles two heads: D % kWidth == 0)
      const uint32_t head = u * kWidth / src.head_dimension;
      if (fp8.k_scale) k_scale = __ldg(fp8.k_scale + head);
      if (fp8.v_scale) v_scale = __ldg(fp8.v_scale + head);
    }
    for (uint32_t t = threadIdx.y; t < kAppendTokens; t += blockDim.y) {
      const uint32_t row = pool_row[t];
      if (row == kSkip) continue;
      const uint64_t from = static_cast<uint64_t>(token[t]) * src.token_stride + static_cast<uint64_t>(u) * kWidth;
      const uint64_t to = static_cast<uint64_t>(row) * src.row_elements + static_cast<uint64_t>(u) * kWidth;
      Unit<kPrec, kWidth> k, v;
      k.load(static_cast<const T *>(src.k) + from);
      v.load(static_cast<const T *>(src.v) + from);
      if constexpr (kFp8) {
        store_e4m3(k, k_scale, static_cast<Out *>(k_pool) + to);
        store_e4m3(v, v_scale, static_cast<Out *>(v_pool) + to);
      } else {
        k.store(static_cast<Out *>(k_pool) + to);
        v.store(static_cast<Out *>(v_pool) + to);
      }
    }
  }
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <int kPrec, int kWidth, bool kFp8>
cudaError_t launch(const PagedKV &pk, const AppendSource &src, void *k_pool, void *v_pool, const Fp8KV &fp8,
                   cudaStream_t stream) {
  const uint32_t units = src.row_elements / kWidth;
  const uint32_t x = units >= kAppendThreads ? kAppendThreads : (units + 31) / 32 * 32;
  const uint32_t y = kAppendThreads / x < kAppendTokens ? kAppendThreads / x : kAppendTokens;
  const dim3 grid((pk.max_row + kAppendTokens - 1) / kAppendTokens, pk.count);
  paged_kv_append<kPrec, kWidth, kFp8><<<grid, dim3(x, y), 0, stream>>>(pk, src, k_pool, v_pool, fp8);
  return cudaGetLastError();
}

// The vector instantiation when every address and stride it touches is aligned to its accesses (16-byte loads; stores
// of 16 bytes, or of kWidth E4M3 bytes), else the scalar one
template <int kPrec>
cudaError_t launch_precision(const PagedKV &pk, const AppendSource &src, void *k_pool, void *v_pool, const Fp8KV *fp8,
                             cudaStream_t stream) {
  constexpr uint32_t bytes = kPrec == FP32 ? 4 : 2;
  const bool sources = aligned16(src.k) && aligned16(src.v) && static_cast<uint64_t>(src.token_stride) * bytes % 16 == 0;
  if (fp8) {
    constexpr int width = 32 / bytes;  // 32 bytes read, `width` bytes written
    const bool pools = (reinterpret_cast<uintptr_t>(k_pool) | reinterpret_cast<uintptr_t>(v_pool)) % width == 0;
    if (sources && pools && src.head_dimension % width == 0)
      return launch<kPrec, width, true>(pk, src, k_pool, v_pool, *fp8, stream);
    return launch<kPrec, 1, true>(pk, src, k_pool, v_pool, *fp8, stream);
  }
  constexpr int width = 16 / bytes;
  if (sources && aligned16(k_pool) && aligned16(v_pool) && static_cast<uint64_t>(src.row_elements) * bytes % 16 == 0)
    return launch<kPrec, width, false>(pk, src, k_pool, v_pool, Fp8KV{}, stream);
  return launch<kPrec, 1, false>(pk, src, k_pool, v_pool, Fp8KV{}, stream);
}

}  // namespace

cudaError_t launch_paged_kv_append(const PagedKV &pk, const AppendSource &src, void *k_pool, void *v_pool,
                                   const Fp8KV *fp8, cudaStream_t stream) {
  switch (src.precision) {
    case FP32: return launch_precision<FP32>(pk, src, k_pool, v_pool, fp8, stream);
    case FP16: return launch_precision<FP16>(pk, src, k_pool, v_pool, fp8, stream);
    default: return launch_precision<BF16>(pk, src, k_pool, v_pool, fp8, stream);
  }
}

}  // namespace mfa
