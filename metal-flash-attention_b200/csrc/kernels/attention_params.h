// Internal launch interface between the C-ABI host layer (csrc/*.cpp) and the sm_90a kernels.
// Not part of the public ABI (include/mfa_b200.h is).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mfa {

// Buffer slots = AttentionOperand.bufferBinding
// (/root/reference/Sources/FlashAttention/Attention/AttentionOperand.swift:52-71).
enum Slot { sQ = 0, sK = 1, sV = 2, sO = 3, sL = 4, sD = 5, sdO = 6, sdV = 7, sdK = 8, sdQ = 9, kSlots = 10 };

// Precision raw values = GEMMOperandPrecision (GEMMOperandPrecision.swift:33-37).
enum Prec : uint8_t { FP32 = 0, FP16 = 1, BF16 = 2 };

struct AttentionParams {
  uint32_t R;      // rows of the attention matrix (output sequence length)
  uint32_t C;      // columns (input sequence length)
  uint32_t D;      // head dimension
  uint32_t batch;  // independent single-head problems, >= 1
  void *buf[kSlots];        // device pointers, by slot
  uint8_t prec[kSlots];     // memory precision, by slot
  uint8_t transposed[kSlots];  // 1: stored [D][seq] (leading dim = seq), 0: [seq][D]
  float scale;       // 1/sqrt(D)          (AttentionKernel+Softmax.swift:17-26)
  float scale_log2;  // log2(e)/sqrt(D)
  // tuning columns of the parameter-table row the kernel was created from (tensor-core family)
  uint8_t exp2_fma_quarters;  // validated and carried; the sm_90a kernels take every exp2 on the MUFU pipe
  uint8_t split_min_blocks;   // 0 = never split small grids
  uint8_t split_max;
};

// compiled exp2-on-the-FMA-pipe variants (quarters of the element pairs): forward 0..2, backward 0..3
constexpr uint32_t kMaxForwardExp2Quarters = 2, kMaxBackwardExp2Quarters = 3;

// ---- SIMT FP32 family (any shape / layout / precision) -------------------------------------
cudaError_t launch_simt_forward(const AttentionParams &p, cudaStream_t stream);
cudaError_t launch_simt_backward_query(const AttentionParams &p, cudaStream_t stream);
cudaError_t launch_simt_backward_key_value(const AttentionParams &p, cudaStream_t stream);
void simt_geometry(int type, uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par, uint32_t *trav,
                   uint32_t *head);

// ---- tensor-core family (wgmma_attention.cu; the backend keeps its historical name "tcgen05" in the ABI) --------
// 16-bit row-major operands with D % 8 == 0 and D <= 256; kernel.cpp stages every other layout into that form.
cudaError_t launch_tcgen05_forward(const AttentionParams &p, cudaStream_t stream);
cudaError_t launch_tcgen05_backward_query(const AttentionParams &p, cudaStream_t stream);
cudaError_t launch_tcgen05_backward_key_value(const AttentionParams &p, cudaStream_t stream);
uint32_t tcgen05_forward_launch_count(uint32_t R, uint32_t C, uint32_t D, uint32_t batch, uint32_t min_blocks,
                                      uint32_t max_splits);
uint32_t tcgen05_backward_launch_count(int type, uint32_t R, uint32_t C, uint32_t D, uint32_t batch, uint32_t min_blocks,
                                       uint32_t max_splits, bool convert_dO);
void tcgen05_forward_set_fused(int enabled);  // debug: 1 = split-KV merged inside the attention kernel (one launch)
void tcgen05_forward_geometry(uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par, uint32_t *trav,
                              uint32_t *head);
void tcgen05_backward_geometry(int type, uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par,
                               uint32_t *trav, uint32_t *head);
bool tcgen05_forward_transposes_ok(uint32_t R, uint32_t C, bool tQ, bool tK, bool tV);
bool tcgen05_backward_transposes_ok(uint32_t R, uint32_t C, bool tQ, bool tK, bool tV, bool tO);

// operand staging for the tensor-core family (pad_head.cu): a [batch][seq][D] (or, transposed, [batch][D][seq]) operand
// is copied to row-major [batch][seq][Dp] with zero padding columns, and an FP32 output computed in that form is copied
// back to the caller's layout
cudaError_t launch_stage_operand(const void *src, void *dst, uint32_t batch, uint32_t seq, uint32_t D, uint32_t Dp,
                                 uint32_t element_bytes, bool transposed, cudaStream_t stream);
cudaError_t launch_unstage_output(const float *src, float *dst, uint32_t batch, uint32_t seq, uint32_t D, uint32_t Dp,
                                  bool transposed, cudaStream_t stream);
cudaError_t launch_bf16_to_f16(const void *src, void *dst, uint64_t elements, cudaStream_t stream);
const char *last_launch_detail();  // thread-local detail string for MFA_ERROR_CUDA messages

}  // namespace mfa
