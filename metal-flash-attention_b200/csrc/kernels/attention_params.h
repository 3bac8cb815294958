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
  // query problems per K/V problem (>= 1, divides batch): query problem b reads K / V problem b / group, and the K, V,
  // dK, dV buffers hold batch / group problems (dK / dV summed over each group)
  uint32_t group;
  void *buf[kSlots];        // device pointers, by slot
  uint8_t prec[kSlots];     // memory precision, by slot
  uint8_t transposed[kSlots];  // 1: stored [D][seq] (leading dim = seq), 0: [seq][D]
  float scale;       // 1/sqrt(D)          (AttentionKernel+Softmax.swift:17-26)
  float scale_log2;  // log2(e)/sqrt(D)
  // tuning columns of the parameter-table row the kernel was created from (tensor-core family)
  uint8_t split_min_blocks;  // 0 = never split small grids
  uint8_t split_max;
  // causal mask, aligned bottom-right: row i sees key j iff j <= i + causal_offset (causal_offset = C - R)
  uint8_t causal;
  int32_t causal_offset;
};

// Packed variable-length sequences (mfa_sequence_table_t), a kernel argument of their own so that the fixed-length
// kernels keep their parameter lists: sequence s owns query rows [row_offsets[s], row_offsets[s + 1]) and key rows
// [column_offsets[s], column_offsets[s + 1]) of every problem, each range clamped into [0, rows] / [0, columns] (the
// rows each problem's buffer holds, AttentionParams R / C).  The grid's z axis is the sequence.
struct Sequences {
  const int32_t *row_offsets, *column_offsets;  // device memory, count + 1 entries each
  uint32_t rows, columns;
  uint32_t count, max_row, max_column;  // host values: they size the grid
};

// The rows of sequence s that a kernel works on, read from the tables and clamped (kernels only)
struct SequenceSpan {
  uint32_t q0, R, k0, C;  // first query row and query count; first key row and key count
};
#ifdef __CUDACC__
// Sequence i's rows in a table: [offsets[i], offsets[i + 1]) clamped into [0, limit], an end below its start empty
__device__ __forceinline__ uint32_t sequence_rows(const int32_t *offsets, uint32_t i, uint32_t limit, uint32_t *first) {
  const int lo = min(max(__ldg(offsets + i), 0), static_cast<int>(limit));
  const int hi = min(max(__ldg(offsets + i + 1), lo), static_cast<int>(limit));
  *first = static_cast<uint32_t>(lo);
  return static_cast<uint32_t>(hi - lo);
}
__device__ __forceinline__ SequenceSpan sequence_span(const Sequences &s, uint32_t i) {
  SequenceSpan r;
  r.R = sequence_rows(s.row_offsets, i, s.rows, &r.q0);
  r.C = sequence_rows(s.column_offsets, i, s.columns, &r.k0);
  return r;
}
#endif

// Paged K/V (mfa_paged_kv_t), the forward's kernel argument: packed query rows as in Sequences, and the keys of
// sequence s in the pages page_table[s][0 .. ceil(Cs / P)) of K / V pools [pages][P][kv_heads][D].
struct PagedKV {
  const int32_t *row_offsets, *column_lengths, *page_table;  // device memory: count + 1, count, count x page_stride
  uint32_t rows;                 // query rows of each problem (AttentionParams R)
  uint32_t pages, page_shift;    // pages in each pool (column / P), log2(P)
  uint32_t page_stride;          // entries per page_table row
  uint32_t max_keys;             // page_stride * P, at most INT32_MAX: no Cs reaches past its page_table row
  uint32_t kv_heads;             // heads of each pool row (batch / group)
  uint32_t count, max_row;       // host values: they size the grid
};
#ifdef __CUDACC__
// Sequence i of a paged call: its query rows (clamped as in sequence_span), k0 = 0 and Cs clamped into [0, max_keys]
__device__ __forceinline__ SequenceSpan paged_span(const PagedKV &pk, uint32_t i) {
  SequenceSpan r;
  r.R = sequence_rows(pk.row_offsets, i, pk.rows, &r.q0);
  r.k0 = 0;
  r.C = static_cast<uint32_t>(min(max(__ldg(pk.column_lengths + i), 0), static_cast<int>(pk.max_keys)));
  return r;
}
// The pool row of key `key` of the sequence whose page_table row is `table` (key < its Cs), the page id clamped into
// [0, pages)
__device__ __forceinline__ uint32_t paged_row(const PagedKV &pk, const int32_t *table, uint32_t key) {
  const int page = min(max(__ldg(table + (key >> pk.page_shift)), 0), static_cast<int>(pk.pages) - 1);
  return (static_cast<uint32_t>(page) << pk.page_shift) | (key & ((1u << pk.page_shift) - 1));
}
#endif

// Sliding-window band (mfa_attention_window_t), a kernel argument of its own so that AttentionParams and the kernels
// without a window keep their parameter lists: row i sees key j iff i + delta - left <= j <= i + delta + right.  The
// host resolves -1 (no bound) and a causal kernel's right (the diagonal) before launch, and clamps both sides to
// min(row + column, INT32_MAX), so the kernels see 0 <= left, right <= INT32_MAX; they add a side to delta or to an
// index in 64 bits.
struct Band {
  int32_t left, right;
};

// FP8 K/V (mfa_fp8_kv_t): the K and V pools of a paged call hold OCP E4M3 bytes, and key row i of K/V head kv stands
// for k_scale[kv] * e4m3(byte) (v_scale for V).  Device arrays of batch / group entries, read by the kernels at launch;
// NULL: every scale is 1.
struct Fp8KV {
  const float *k_scale, *v_scale;
};

// Paged K/V append (mfa_paged_kv_append_t): the step's new tokens, token t's K/V head kv, element d at element
// t * token_stride + kv * D + d of k / v, in `precision`
struct AppendSource {
  const void *k, *v;
  uint32_t token_stride;   // elements, >= row_elements
  uint32_t head_dimension; // D
  uint32_t row_elements;   // kv_heads * D: the elements of one pool row
  uint8_t precision;       // Prec
};
// The append of paged_kv_append.cu: one launch, grid (tokens of max_row, count).  fp8: the pools hold E4M3 bytes
// quantized with its scales; nullptr: the pools hold `precision` elements, copied bit for bit
cudaError_t launch_paged_kv_append(const PagedKV &pk, const AppendSource &src, void *k_pool, void *v_pool,
                                   const Fp8KV *fp8, cudaStream_t stream);

// Rotary append (mfa_rotary_t): the step's queries, token t's query head h, element d at t * q_token_stride + h * D + d
// of q, in the append's precision, rotated into q_out [query_heads][rows][D]; cos / sin FP32, position p, frequency j
// at p * table_stride + j
struct RotarySource {
  const void *q;
  void *q_out;
  const float *cos, *sin;
  uint32_t query_heads;
  uint32_t q_token_stride;  // elements, >= query_heads * D
  uint32_t rotary_dim;      // r: even, 2..D
  uint32_t table_stride;    // floats, >= r / 2
  bool interleaved;         // pairs (2j, 2j + 1), else (j, j + r / 2)
};
// The rotary append of rotary_append.cu: the append above, with q and k rotated at their cache positions, in one launch
cudaError_t launch_rotary_kv_append(const PagedKV &pk, const AppendSource &src, const RotarySource &rot, void *k_pool,
                                    void *v_pool, const Fp8KV *fp8, cudaStream_t stream);

// The form of a call: fixed-length problems, or packed sequences (seq) or a paged cache (pk); a window; FP8 pools
// (paged); a split-KV request of a packed or paged call (num_splits 0: the plan's choice; key_bound: every Cs's bound).
// The backward takes seq and band only: the host rejects a paged table, a split and FP8 for any kernel but the forward.
struct AttentionCall {
  const Sequences *seq = nullptr;
  const PagedKV *pk = nullptr;
  const Band *band = nullptr;
  const Fp8KV *fp8 = nullptr;
  bool split = false;
  uint32_t num_splits = 0, key_bound = 0;
};

// ---- SIMT FP32 family (any shape / layout / precision) -------------------------------------
// Kernel `type` (mfa_kernel_type_t) in the form of call.seq, call.pk and call.band (a null one: absent), never split;
// FP8 K/V is not served here
cudaError_t launch_simt(int type, const AttentionParams &p, const AttentionCall &call, cudaStream_t stream);
void simt_geometry(int type, uint32_t D, uint32_t *threads, uint32_t *smem_bytes, uint32_t *par, uint32_t *trav,
                   uint32_t *head);

// ---- tensor-core family (wgmma_attention.cu; the backend keeps its historical name "tcgen05" in the ABI) --------
// 16-bit row-major operands with D % 8 == 0 and D <= kWgmmaMaxHead; kernel.cpp stages every other layout into that form.
constexpr uint32_t kWgmmaMaxHead = 256;
// Kernel `type` (mfa_kernel_type_t) in the form of `call`, on the grid of its wgmma_plan
cudaError_t launch_wgmma(int type, const AttentionParams &p, const AttentionCall &call, cudaStream_t stream);
// How the launcher of kernel `type` (mfa_kernel_type_t) runs one problem of padded head dimension D; every field is
// derived from the kernels' compile-time configurations.  R, C and batch do not affect the geometry fields.
struct WgmmaPlan {
  uint32_t threads, smem_bytes;        // per CTA
  uint32_t par, trav, head;            // blockDimensions: rows per CTA, rows per pipeline stage, head block
  dim3 grid;                           // (tiles, batch, splits); dK/dV: (tiles, batch / group, splits)
  uint32_t blocks_per_split, splits;   // traversal blocks per CTA; ranges of the traversal axis (1 = not split)
  bool convert_dO_first;               // dK/dV: the BF16 dO is converted to FP16 in a pass of its own
  uint32_t launches;                   // kernels the launcher issues
  uint32_t heads_per_tile;             // split-KV packed / paged forward: query heads per tile (1 elsewhere)
};
// The plan of a call of kernel `type`, which its launcher and the host's counts follow.  batch = query problems,
// group = query problems per K/V problem (only the dK/dV plan, whose CTAs own K/V tiles, and the split-KV forward
// depend on it); min_blocks and max_splits: the parameter-table row's tuning columns; convert_dO: BF16 dO beside FP16
// Q/K/V (only the dK/dV plan depends on it).
// - Fixed-length problems: grid (tiles, heads, splits), the traversal axis split only when the SMs would otherwise
//   idle.  call.band (host-resolved, as launched): only the band's width in traversal blocks is what the split cuts.
// - Packed sequences or a paged cache, unsplit: never split, grid (tiles of the longest sequence, heads, count); the
//   dO-conversion choice counts every CTA of that grid.
// - A split-KV packed or paged forward (mfa_split_plan_t), unless it plans one split and one head per tile: grid (tiles
//   of max_row x splits, batch / heads_per_tile, count).  call.key_bound bounds every sequence's keys; num_splits 0
//   lets the tuning columns choose over ceil(key_bound / BN) blocks (a window's band width when narrower);
//   heads_per_tile: the group (2..128) when max_row < 128, so that a tile holds 128 / group rows of each query head of
//   a K/V head.
// An empty call gives the geometry fields, which depend on neither the problem size nor the device.
WgmmaPlan wgmma_plan(int type, uint32_t D, uint32_t R, uint32_t C, uint32_t batch, uint32_t group, uint32_t min_blocks,
                     uint32_t max_splits, bool convert_dO, const AttentionCall &call, uint32_t sm_count);

// operand staging for the tensor-core family (pad_head.cu): a [batch][seq][D] (or, transposed, [batch][D][seq]) operand
// is copied to row-major [batch][seq][Dp] with zero padding columns, and an FP32 output computed in that form is copied
// back to the caller's layout
cudaError_t launch_stage_operand(const void *src, void *dst, uint32_t batch, uint32_t seq, uint32_t D, uint32_t Dp,
                                 uint32_t element_bytes, bool transposed, cudaStream_t stream);
cudaError_t launch_unstage_output(const float *src, float *dst, uint32_t batch, uint32_t seq, uint32_t D, uint32_t Dp,
                                  bool transposed, cudaStream_t stream);
// packed sequences: only rows [0, min(length, limit)) of each of the `count` sequences of `offsets` (the rows the
// attention kernels wrote), so that rows outside every sequence keep the caller's contents
cudaError_t launch_unstage_sequences(const float *src, float *dst, uint32_t batch, uint32_t seq, const int32_t *offsets,
                                     uint32_t count, uint32_t limit, uint32_t D, uint32_t Dp, bool transposed,
                                     cudaStream_t stream);
cudaError_t launch_bf16_to_f16(const void *src, void *dst, uint64_t elements, cudaStream_t stream);
const char *last_launch_detail();  // thread-local detail string for MFA_ERROR_CUDA messages

}  // namespace mfa
