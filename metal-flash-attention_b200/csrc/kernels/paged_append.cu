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

#include "append_common.cuh"

namespace mfa {
namespace {

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
