// Rotary append (mfa_paged_kv_append_rotary): the paged K/V append of paged_append.cu, with the step's queries and new
// keys rotated by RoPE at their cache positions, and the queries written in the paged forward's [H][rows][D] layout.
// New token i of sequence s is at position p = Cs - Rs + i (the key the plain append writes); pair (x, y) of every query
// head and every K/V head becomes (x c - y s, y c + x s) with c = cos[p][j], s = sin[p][j], each product and the sum
// rounded separately (no FMA), then rounded to the source precision; V is appended as the plain append does.
//
// One CTA per (kAppendTokens tokens, sequence): its first threads resolve each token's position and pool row once, then
// threadIdx.x walks the items of a token and threadIdx.y the tokens.  An item is a unit of kWidth frequencies (a vector
// of the x elements and one of the y elements) or of kWidth pass-through elements (d >= r) of kHeadChunk consecutive
// heads of the concatenated query and key heads, so each table entry is read once per chunk; or one unit of V.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "append_common.cuh"

namespace mfa {
namespace {

// heads per item: the table entries of a unit are read once per chunk.  One head for E4M3 pools, whose IEEE divisions
// call a slow path: table entries kept across those calls spill
template <bool kFp8>
constexpr uint32_t kHeadChunk = kFp8 ? 1 : 4;

// x rounded to nearest-even into the unit's element j (FP32: x itself)
template <int kPrec, int kWidth>
__device__ __forceinline__ void set(Unit<kPrec, kWidth> &u, int j, float x) {
  uint32_t *w = reinterpret_cast<uint32_t *>(u.v);
  if constexpr (kPrec == FP32) {
    w[j] = __float_as_uint(x);
  } else {
    const uint32_t bits = kPrec == BF16 ? static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16_rn(x)))
                                        : static_cast<uint32_t>(__half_as_ushort(__float2half_rn(x)));
    const int shift = 16 * (j % 2);
    w[j / 2] = (w[j / 2] & ~(0xffffu << shift)) | (bits << shift);
  }
}
// element e of the 2 kWidth elements x then y
template <int kPrec, int kWidth>
__device__ __forceinline__ void set_pair_element(Unit<kPrec, kWidth> &x, Unit<kPrec, kWidth> &y, int e, float v) {
  if (e < kWidth)
    set(x, e, v);
  else
    set(y, e - kWidth, v);
}

// grid (ceil(max_row / kAppendTokens), count), block (items of a token, up to 256 threads; tokens)
template <int kPrec, int kWidth, bool kFp8, bool kInterleaved>
__global__ void __launch_bounds__(kAppendThreads)
    rotary_kv_append(const PagedKV pk, const AppendSource src, const RotarySource rot, void *__restrict__ k_pool,
                     void *__restrict__ v_pool, const Fp8KV fp8) {
  using T = typename Element<kPrec>::T;
  using Out = typename std::conditional<kFp8, uint8_t, T>::type;
  __shared__ uint32_t pool_row[kAppendTokens], position[kAppendTokens], token[kAppendTokens];
  const uint32_t s = blockIdx.y;
  if (threadIdx.y == 0 && threadIdx.x < kAppendTokens) {
    const SequenceSpan span = paged_span(pk, s);
    const uint32_t i = blockIdx.x * kAppendTokens + threadIdx.x;
    uint32_t p = kSkip;
    pool_row[threadIdx.x] = token_slot(pk, span, s, i, &p);
    position[threadIdx.x] = p;
    token[threadIdx.x] = span.q0 + i;
  }
  __syncthreads();
  const uint32_t D = src.head_dimension, H = rot.query_heads, heads = H + pk.kv_heads;
  const uint32_t half = rot.rotary_dim / 2;
  const uint32_t rotary_units = half / kWidth;  // (the host picks kWidth > 1 only when it divides r / 2 and D)
  const uint32_t head_units = rotary_units + (D - rot.rotary_dim) / kWidth;
  const uint32_t head_items = head_units * ((heads + kHeadChunk<kFp8> - 1) / kHeadChunk<kFp8>);
  const uint32_t items = head_items + src.row_elements / kWidth;
  for (uint32_t u = threadIdx.x; u < items; u += blockDim.x) {
    for (uint32_t t = threadIdx.y; t < kAppendTokens; t += blockDim.y) {
      const uint32_t p = position[t], row = pool_row[t];
      if (p == kSkip) continue;
      const uint64_t from = static_cast<uint64_t>(token[t]) * src.token_stride;
      const uint64_t to = static_cast<uint64_t>(row) * src.row_elements;
      if (u >= head_items) {  // a unit of V, as the plain append writes it
        if (row == kSkip) continue;
        const uint32_t e = (u - head_items) * kWidth;
        Unit<kPrec, kWidth> v;
        v.load(static_cast<const T *>(src.v) + from + e);
        if constexpr (kFp8) {
          store_e4m3(v, fp8.v_scale ? __ldg(fp8.v_scale + e / D) : 1.0f, static_cast<Out *>(v_pool) + to + e);
        } else {
          v.store(static_cast<Out *>(v_pool) + to + e);
        }
        continue;
      }
      const uint32_t unit = u % head_units, h0 = u / head_units * kHeadChunk<kFp8>;
      const bool rotary = unit < rotary_units;
      // the unit's elements: a (and b, for a rotary unit) within a head
      const uint32_t j0 = unit * kWidth;
      const uint32_t a = !rotary ? rot.rotary_dim + (unit - rotary_units) * kWidth : kInterleaved ? 2 * j0 : j0;
      const uint32_t b = kInterleaved ? a + kWidth : a + half;
      float c[kWidth], sn[kWidth];
      if (rotary) {
        const uint64_t entry = static_cast<uint64_t>(p) * rot.table_stride + j0;
#pragma unroll
        for (int k = 0; k < kWidth; ++k) {
          c[k] = __ldg(rot.cos + entry + k);
          sn[k] = __ldg(rot.sin + entry + k);
        }
      }
      const uint64_t q_from = static_cast<uint64_t>(token[t]) * rot.q_token_stride;
#pragma unroll
      for (uint32_t n = 0; n < kHeadChunk<kFp8>; ++n) {
        const uint32_t h = h0 + n;
        if (h >= heads) break;
        const bool query = h < H;
        if (!query && row == kSkip) break;  // (key heads follow every query head)
        const T *in = query ? static_cast<const T *>(rot.q) + q_from + static_cast<uint64_t>(h) * D
                            : static_cast<const T *>(src.k) + from + static_cast<uint64_t>(h - H) * D;
        Unit<kPrec, kWidth> x, y;
        x.load(in + a);
        if (rotary) {
          y.load(in + b);
          float fx[2 * kWidth];
#pragma unroll
          for (int k = 0; k < kWidth; ++k) {
            fx[k] = x.at(k);
            fx[kWidth + k] = y.at(k);
          }
          // pair k: NeoX (x_k, y_k); interleaved, elements 2k and 2k + 1 of the 2 kWidth elements x then y
#pragma unroll
          for (int k = 0; k < kWidth; ++k) {
            const float xv = kInterleaved ? fx[2 * k] : fx[k], yv = kInterleaved ? fx[2 * k + 1] : fx[kWidth + k];
            const float xr = __fsub_rn(__fmul_rn(xv, c[k]), __fmul_rn(yv, sn[k]));
            const float yr = __fadd_rn(__fmul_rn(yv, c[k]), __fmul_rn(xv, sn[k]));
            if constexpr (kInterleaved) {
              set_pair_element(x, y, 2 * k, xr);
              set_pair_element(x, y, 2 * k + 1, yr);
            } else {
              set(x, k, xr);
              set(y, k, yr);
            }
          }
        }
        if (query) {
          T *out = static_cast<T *>(rot.q_out) + (static_cast<uint64_t>(h) * pk.rows + token[t]) * D;
          x.store(out + a);
          if (rotary) y.store(out + b);
        } else if constexpr (kFp8) {
          const float scale = fp8.k_scale ? __ldg(fp8.k_scale + (h - H)) : 1.0f;
          Out *out = static_cast<Out *>(k_pool) + to + static_cast<uint64_t>(h - H) * D;
          store_e4m3(x, scale, out + a);
          if (rotary) store_e4m3(y, scale, out + b);
        } else {
          Out *out = static_cast<Out *>(k_pool) + to + static_cast<uint64_t>(h - H) * D;
          x.store(out + a);
          if (rotary) y.store(out + b);
        }
      }
    }
  }
}

template <int kPrec, int kWidth, bool kFp8, bool kInterleaved>
cudaError_t launch(const PagedKV &pk, const AppendSource &src, const RotarySource &rot, void *k_pool, void *v_pool,
                   const Fp8KV &fp8, cudaStream_t stream) {
  const uint32_t heads = rot.query_heads + pk.kv_heads;
  const uint32_t head_units = rot.rotary_dim / 2 / kWidth + (src.head_dimension - rot.rotary_dim) / kWidth;
  const uint32_t items = head_units * ((heads + kHeadChunk<kFp8> - 1) / kHeadChunk<kFp8>) + src.row_elements / kWidth;
  const uint32_t x = items >= kAppendThreads ? kAppendThreads : (items + 31) / 32 * 32;
  const uint32_t y = kAppendThreads / x < kAppendTokens ? kAppendThreads / x : kAppendTokens;
  const dim3 grid((pk.max_row + kAppendTokens - 1) / kAppendTokens, pk.count);
  rotary_kv_append<kPrec, kWidth, kFp8, kInterleaved>
      <<<grid, dim3(x, y), 0, stream>>>(pk, src, rot, k_pool, v_pool, fp8);
  return cudaGetLastError();
}

template <int kPrec, bool kInterleaved>
cudaError_t launch_pairing(const PagedKV &pk, const AppendSource &src, const RotarySource &rot, void *k_pool,
                           void *v_pool, const Fp8KV *fp8, cudaStream_t stream) {
  constexpr uint32_t bytes = kPrec == FP32 ? 4 : 2;
  // the vector instantiation when every address and stride it touches is aligned to its accesses and a unit never
  // straddles a head, the rotary boundary or its pair's half (kWidth divides D and r / 2), else the scalar one
  const auto vector = [&](uint32_t width, bool pools) {
    return pools && aligned16(src.k) && aligned16(src.v) && aligned16(rot.q) && aligned16(rot.q_out) &&
           static_cast<uint64_t>(src.token_stride) * bytes % 16 == 0 &&
           static_cast<uint64_t>(rot.q_token_stride) * bytes % 16 == 0 && src.head_dimension % width == 0 &&
           rot.rotary_dim / 2 % width == 0;
  };
  if (fp8) {
    constexpr int width = 32 / bytes;  // 32 bytes read, `width` bytes written
    if (vector(width, (reinterpret_cast<uintptr_t>(k_pool) | reinterpret_cast<uintptr_t>(v_pool)) % width == 0))
      return launch<kPrec, width, true, kInterleaved>(pk, src, rot, k_pool, v_pool, *fp8, stream);
    return launch<kPrec, 1, true, kInterleaved>(pk, src, rot, k_pool, v_pool, *fp8, stream);
  }
  constexpr int width = 16 / bytes;
  if (vector(width, aligned16(k_pool) && aligned16(v_pool)))
    return launch<kPrec, width, false, kInterleaved>(pk, src, rot, k_pool, v_pool, Fp8KV{}, stream);
  return launch<kPrec, 1, false, kInterleaved>(pk, src, rot, k_pool, v_pool, Fp8KV{}, stream);
}

template <int kPrec>
cudaError_t launch_precision(const PagedKV &pk, const AppendSource &src, const RotarySource &rot, void *k_pool,
                             void *v_pool, const Fp8KV *fp8, cudaStream_t stream) {
  return rot.interleaved ? launch_pairing<kPrec, true>(pk, src, rot, k_pool, v_pool, fp8, stream)
                         : launch_pairing<kPrec, false>(pk, src, rot, k_pool, v_pool, fp8, stream);
}

}  // namespace

cudaError_t launch_rotary_kv_append(const PagedKV &pk, const AppendSource &src, const RotarySource &rot, void *k_pool,
                                    void *v_pool, const Fp8KV *fp8, cudaStream_t stream) {
  switch (src.precision) {
    case FP32: return launch_precision<FP32>(pk, src, rot, k_pool, v_pool, fp8, stream);
    case FP16: return launch_precision<FP16>(pk, src, rot, k_pool, v_pool, fp8, stream);
    default: return launch_precision<BF16>(pk, src, rot, k_pool, v_pool, fp8, stream);
  }
}

}  // namespace mfa
