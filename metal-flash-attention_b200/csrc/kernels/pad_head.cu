// Operand staging for the tensor-core family.  TMA needs a 16-byte row pitch, i.e. D % 8 == 0 for 16-bit operands; the
// reference covers any D by zero-padding inside its async copies (AttentionKernel+OuterProduct.swift:237-254,
// GEMMHeaders.swift:111-114).  Here an operand whose head dimension is not a multiple of 8, or that is stored transposed
// ([D][seq]), is copied once into a row-major staging buffer with pad8(D) columns (zeros in the padding -- exact: every
// contraction over D only gains zero terms), the wgmma kernels run on the staged operands, and the FP32 outputs are copied
// back to the caller's layout without the padding.  The copies are O(N D)
// against O(N^2 D) of attention work: D = 35, 77, 95, 199 (the reference's own test shapes,
// SquareAttentionTest.swift:6-25) run on the tensor cores instead of the FP32 CUDA-core family.
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_params.h"
#include "backward_common.cuh"

namespace mfa {
namespace {

// dst[b][s][c] = c < D ? src(b, s, c) : 0 for c < Dp, src row-major [b][s][D] or transposed [b][D][s]; one thread per
// destination element
template <typename T>
__global__ void __launch_bounds__(256) stage_operand(const T *__restrict__ src, T *__restrict__ dst, uint32_t seq, uint32_t D,
                                                     uint32_t Dp, uint64_t total, bool transposed) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const uint64_t row = i / Dp;  // b * seq + s
  const uint32_t c = static_cast<uint32_t>(i % Dp);
  const uint64_t b = row / seq, s = row % seq;
  dst[i] = c < D ? src[transposed ? (b * D + c) * seq + s : row * D + c] : T(0);
}

// dst(b, s, c) = src[b][s][c] for c < D (src has Dp columns); one thread per destination element, in dst order
__global__ void __launch_bounds__(256) unstage_output(const float *__restrict__ src, float *__restrict__ dst, uint32_t seq,
                                                      uint32_t D, uint32_t Dp, uint64_t total, bool transposed) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  uint64_t b, s, c;
  if (transposed) {  // dst [b][D][seq]
    s = i % seq;
    c = (i / seq) % D;
    b = i / (static_cast<uint64_t>(seq) * D);
  } else {
    c = i % D;
    s = (i / D) % seq;
    b = i / (static_cast<uint64_t>(seq) * D);
  }
  dst[i] = src[(b * seq + s) * Dp + c];
}

// Packed sequences: unstage_output of only the rows the attention kernels wrote, rows [0, min(length, limit)) of
// sequence blockIdx.z (its range in `offsets`, clamped into [0, seq] as the kernels clamp it) of problem blockIdx.y
__global__ void __launch_bounds__(256) unstage_sequences(const float *__restrict__ src, float *__restrict__ dst,
                                                         const int32_t *__restrict__ offsets, uint32_t seq,
                                                         uint32_t limit, uint32_t D, uint32_t Dp, bool transposed) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  uint32_t first;
  const uint32_t rows = min(sequence_rows(offsets, blockIdx.z, seq, &first), limit);
  if (i >= static_cast<uint64_t>(rows) * D) return;
  const uint64_t b = blockIdx.y, s = first + i / D, c = i % D;
  dst[transposed ? (b * D + c) * seq + s : (b * seq + s) * D + c] = src[(b * seq + s) * Dp + c];
}

// dO (BF16) -> FP16, eight elements per thread; exact for 2^-14 <= |x| < 65504 (backward_common.cuh)
__global__ void __launch_bounds__(256) bf16_to_f16(const uint4 *__restrict__ src, uint4 *__restrict__ dst, uint64_t vectors) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < vectors) dst[i] = bwd::bf16x8_to_f16x8(src[i]);
}

}  // namespace

cudaError_t launch_bf16_to_f16(const void *src, void *dst, uint64_t elements, cudaStream_t stream) {
  const uint64_t vectors = elements / 8;  // D % 8 == 0
  bf16_to_f16<<<static_cast<uint32_t>((vectors + 255) / 256), 256, 0, stream>>>(static_cast<const uint4 *>(src),
                                                                                 static_cast<uint4 *>(dst), vectors);
  return cudaGetLastError();
}

cudaError_t launch_stage_operand(const void *src, void *dst, uint32_t batch, uint32_t seq, uint32_t D, uint32_t Dp,
                                 uint32_t element_bytes, bool transposed, cudaStream_t stream) {
  const uint64_t n = static_cast<uint64_t>(batch) * seq * Dp;
  const uint32_t blocks = static_cast<uint32_t>((n + 255) / 256);
  if (element_bytes == 2)
    stage_operand<uint16_t><<<blocks, 256, 0, stream>>>(static_cast<const uint16_t *>(src), static_cast<uint16_t *>(dst), seq,
                                                        D, Dp, n, transposed);
  else
    stage_operand<uint32_t><<<blocks, 256, 0, stream>>>(static_cast<const uint32_t *>(src), static_cast<uint32_t *>(dst), seq,
                                                        D, Dp, n, transposed);
  return cudaGetLastError();
}

cudaError_t launch_unstage_output(const float *src, float *dst, uint32_t batch, uint32_t seq, uint32_t D, uint32_t Dp,
                                  bool transposed, cudaStream_t stream) {
  const uint64_t n = static_cast<uint64_t>(batch) * seq * D;
  unstage_output<<<static_cast<uint32_t>((n + 255) / 256), 256, 0, stream>>>(src, dst, seq, D, Dp, n, transposed);
  return cudaGetLastError();
}

cudaError_t launch_unstage_sequences(const float *src, float *dst, uint32_t batch, uint32_t seq, const int32_t *offsets,
                                     uint32_t count, uint32_t limit, uint32_t D, uint32_t Dp, bool transposed,
                                     cudaStream_t stream) {
  const uint64_t n = static_cast<uint64_t>(limit) * D;
  unstage_sequences<<<dim3(static_cast<uint32_t>((n + 255) / 256), batch, count), 256, 0, stream>>>(
      src, dst, offsets, seq, limit, D, Dp, transposed);
  return cudaGetLastError();
}

}  // namespace mfa
