// AttentionKernel side of the C ABI: handle creation/validation, launch geometry, and encode()
// -- the compile + bind + dispatch the reference leaves to its caller
// (Tests/FlashAttentionTests/Attention/SquareAttentionTest.swift:240-372).
// Mirrors Sources/FlashAttention/Attention/AttentionKernel/AttentionKernel.swift.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "internal.h"
#include "kernels/device_state.h"

struct mfa_attention_kernel {
  mfa_attention_kernel_descriptor_t descriptor;
  int type;
  int backend;
  uint32_t threads, smem_bytes, par, trav, head;
  std::string source_name;
  bool windowed;                   // mfa_attention_kernel_create_windowed
  mfa_attention_window_t window;   // as given (-1: no bound on that side)
};

namespace mfa {

// loadFunction / storeFunction legality (AttentionKernel.swift:81-139): a 16-bit memory format may
// only be widened to FP32 or kept as is; FP32 memory can only be FP32 in registers.
static bool precision_pair_valid(int memory, int reg) {
  if (memory == MFA_FP16) return reg == MFA_FP16 || reg == MFA_FP32;
  if (memory == MFA_BF16) return reg == MFA_BF16 || reg == MFA_FP32;
  if (memory == MFA_FP32) return reg == MFA_FP32;
  return false;
}

static const int *operands_of(int type, int *count) {
  static const int fwd[] = {MFA_Q, MFA_K, MFA_V, MFA_O, MFA_L};
  static const int dq[] = {MFA_Q, MFA_K, MFA_V, MFA_O, MFA_L, MFA_D, MFA_dO, MFA_dQ};
  static const int dkv[] = {MFA_Q, MFA_K, MFA_V, MFA_L, MFA_D, MFA_dO, MFA_dV, MFA_dK};
  switch (type) {
    case MFA_FORWARD: *count = 5; return fwd;
    case MFA_BACKWARD_QUERY: *count = 8; return dq;
    default: *count = 8; return dkv;
  }
}

static bool is_output(int type, int slot) {
  return type == MFA_FORWARD ? slot == MFA_O : (type == MFA_BACKWARD_QUERY ? slot == MFA_dQ : (slot == MFA_dV || slot == MFA_dK));
}

// The operands (bit = buffer slot) the tensor-core family copies into a row-major, pad8(D)-column staging buffer: every
// operand with a head dimension when D % 8 != 0, and any operand stored transposed (L and D are per-row vectors, never
// staged).  encode() stages each input and copies each output back: one launch apiece.
static uint32_t staged_operands(const mfa_attention_kernel *k) {
  if (k->backend != MFA_BACKEND_TCGEN05) return 0;
  const bool padded = k->descriptor.head_dimension % 8 != 0;
  uint32_t mask = 0;
  int n = 0;
  const int *ops = operands_of(k->type, &n);
  for (int i = 0; i < n; ++i)
    if (ops[i] != MFA_L && ops[i] != MFA_D && (padded || ((k->descriptor.transpose_state_mask >> ops[i]) & 1)))
      mask |= 1u << ops[i];
  return mask;
}

// Several kernels carry the batch in gridDim.y (limit 65535; the SIMT dK/dV kernel multiplies it by up to four head
// slices): larger batches go out as several launches over slices of the batch -- the problems are independent and
// stored back to back, so a slice is just a pointer offset.  With grouped K/V every slice holds whole groups (its K/V
// problems start at h0 / group), so a dK/dV CTA still sums over all query problems of its group.  Calls f(first
// problem, problems) per slice and stops at the first status other than MFA_SUCCESS.
constexpr uint32_t kMaxBatchPerLaunch = 16384;
template <class F>
static int for_each_batch_slice(uint32_t batch, uint32_t group, F f) {
  const uint32_t step = kMaxBatchPerLaunch / group * group;
  for (uint32_t h0 = 0; h0 < batch; h0 += step) {
    const int status = f(h0, batch - h0 < step ? batch - h0 : step);
    if (status != MFA_SUCCESS) return status;
  }
  return MFA_SUCCESS;
}

// The query problems per K/V problem of the launch constants (kv_group 0 or 1: every problem has its own K and V)
static int kv_group_of(const mfa_function_constants_t *c, uint32_t *group) {
  const uint32_t batch = c->batch_count ? c->batch_count : 1, g = c->kv_group ? c->kv_group : 1;
  if (g > kMaxBatchPerLaunch)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "kv_group " + std::to_string(g) + " exceeds " +
                                                std::to_string(kMaxBatchPerLaunch) +
                                                ", the query problems of one launch slice.");
  if (batch % g != 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "batch_count " + std::to_string(batch) + " is not a multiple of kv_group " +
                                                std::to_string(g) + ".");
  *group = g;
  return MFA_SUCCESS;
}

static bool key_value_slot(int slot) { return slot == sK || slot == sV || slot == sdK || slot == sdV; }

// sm_90 check of the current device, cached per device ordinal (encode() of a microsecond-scale kernel must not pay
// two runtime queries per call)
static int check_device() {
  const int device = current_device();
  if (device < 0)
    return fail(MFA_ERROR_NO_DEVICE, "No CUDA device (cudaGetDevice failed; this library has no CPU fallback).");
  static std::mutex mutex;
  static int8_t verdict[kMaxDevices] = {};  // 0 unknown, 1 sm_90, -1 other
  if (device < kMaxDevices) {
    std::lock_guard<std::mutex> lock(mutex);
    if (verdict[device] == 1) return MFA_SUCCESS;
  }
  int major = 0;
  cudaError_t e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
  if (e != cudaSuccess) return fail(MFA_ERROR_NO_DEVICE, std::string("cudaDeviceGetAttribute: ") + cudaGetErrorString(e));
  if (major != 9)
    return fail(MFA_ERROR_NO_DEVICE, "Device is not sm_90 (compute capability " + std::to_string(major) +
                                         ".x); these kernels are built for sm_90a only.");
  if (device < kMaxDevices) {
    std::lock_guard<std::mutex> lock(mutex);
    verdict[device] = 1;
  }
  return MFA_SUCCESS;
}

static int build_params(const mfa_attention_kernel *k, const mfa_function_constants_t *c, void *const buffers[],
                        AttentionParams &p) {
  if (c->row == 0 || c->column == 0) return fail(MFA_ERROR_INVALID_ARGUMENT, "R and C must be at least 1.");
  p.R = c->row;
  p.C = c->column;
  p.D = k->descriptor.head_dimension;
  p.batch = c->batch_count ? c->batch_count : 1;
  const int status = kv_group_of(c, &p.group);
  if (status != MFA_SUCCESS) return status;
  for (int s = 0; s < kSlots; ++s) {
    p.buf[s] = buffers[s];
    uint8_t mp = k->descriptor.memory_precisions[s];
    p.prec[s] = mp == 0xFF ? 0 : mp;
    p.transposed[s] = (k->descriptor.transpose_state_mask >> s) & 1;
  }
  // dotProductScale (AttentionKernel+Softmax.swift:17-26)
  p.scale = 1.0f / std::sqrt(static_cast<float>(p.D));
  p.scale_log2 = 1.442695041f * p.scale;
  // the tuning columns of the parameter-table row this kernel was created from
  p.split_min_blocks = k->descriptor.split_min_blocks;
  p.split_max = k->descriptor.split_max ? k->descriptor.split_max : 1;
  p.causal = k->descriptor.causal;
  p.causal_offset = static_cast<int32_t>(static_cast<int64_t>(p.C) - static_cast<int64_t>(p.R));
  int n = 0;
  const int *ops = operands_of(k->type, &n);
  for (int i = 0; i < n; ++i)
    if (buffers[ops[i]] == nullptr)
      return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Buffer ") + mfa_operand_name((mfa_operand_t)ops[i]) +
                                                  " (binding " + std::to_string(ops[i]) + ") is NULL.");
  return MFA_SUCCESS;
}

// The band a windowed kernel launches with over problems (or sequences) of at most `rows` x `columns`: -1 and anything
// above rows + columns (which no band can exceed) become rows + columns, capped at INT32_MAX, and a causal kernel's
// right side is the diagonal.  nullptr for a kernel without a window.
static const Band *band_of(const mfa_attention_kernel *k, uint64_t rows, uint64_t columns, Band *out) {
  if (!k->windowed) return nullptr;
  const int64_t limit = static_cast<int64_t>(std::min<uint64_t>(rows + columns, 0x7fffffffu));
  auto side = [&](int32_t v) { return static_cast<int32_t>(v < 0 || v > limit ? limit : v); };
  *out = Band{side(k->window.left), k->descriptor.causal ? 0 : side(k->window.right)};
  return out;
}

// The launch form of a packed-sequence table, after the checks the host can make without reading device memory
constexpr uint32_t kMaxSequences = 65535;  // the grid's z limit
static int sequences_of(const mfa_attention_kernel *k, const mfa_function_constants_t *c, const mfa_sequence_table_t *t,
                        Sequences *out) {
  if (!t) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL sequence table.");
  // (the tensor-core family stages transposed operands row-major; the SIMT packed kernels read row-major operands only)
  if (k->backend == MFA_BACKEND_SIMT_FP32) {
    int n = 0;
    const int *ops = operands_of(k->type, &n);
    for (int i = 0; i < n; ++i)
      if ((k->descriptor.transpose_state_mask >> ops[i]) & 1)
        return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Packed sequences on MFA_BACKEND_SIMT_FP32 need row-major "
                                                            "operands; ") +
                                                    mfa_operand_name((mfa_operand_t)ops[i]) + " is transposed.");
  }
  if (!t->row_offsets || !t->column_offsets)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Sequence table: row_offsets and column_offsets must not be NULL.");
  if (t->count == 0 || t->count > kMaxSequences)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Sequence table: count " + std::to_string(t->count) +
                                                " is outside [1, " + std::to_string(kMaxSequences) + "].");
  if (t->max_row == 0 || t->max_row > c->row)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Sequence table: max_row " + std::to_string(t->max_row) +
                                                " is outside [1, row = " + std::to_string(c->row) + "].");
  if (t->max_column == 0 || t->max_column > c->column)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Sequence table: max_column " + std::to_string(t->max_column) +
                                                " is outside [1, column = " + std::to_string(c->column) + "].");
  *out = Sequences{t->row_offsets, t->column_offsets, c->row, c->column, t->count, t->max_row, t->max_column};
  return MFA_SUCCESS;
}

// The launch form of a paged K/V table's own fields, after the checks the host can make without reading device memory,
// shared by the forward and the append: the queries (new tokens) are `rows` rows of their buffer and the pools
// `columns` rows.  rows_name / columns_name: what the messages call them.  kv_heads is left for the caller.
static int paged_table_of(const mfa_paged_kv_t *t, uint32_t rows, uint32_t columns, const char *rows_name,
                          const char *columns_name, PagedKV *out) {
  if (!t->row_offsets || !t->column_lengths || !t->page_table)
    return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Paged K/V: ") +
                                                (!t->row_offsets ? "row_offsets" : !t->column_lengths ? "column_lengths"
                                                                                                      : "page_table") +
                                                " must not be NULL.");
  if (t->count == 0 || t->count > kMaxSequences)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V: count " + std::to_string(t->count) + " is outside [1, " +
                                                std::to_string(kMaxSequences) + "].");
  if (t->max_row == 0 || t->max_row > rows)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V: max_row " + std::to_string(t->max_row) + " is outside [1, " +
                                                rows_name + " = " + std::to_string(rows) + "].");
  const uint32_t P = t->page_size;
  if (P < 16 || (P & (P - 1)) != 0 || columns % P != 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V: page_size " + std::to_string(P) +
                                                " must be a power of two, at least 16, dividing " + columns_name + " = " +
                                                std::to_string(columns) + ".");
  if (t->page_stride == 0) return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V: page_stride 0 must be at least 1.");
  uint32_t shift = 0;
  while ((1u << shift) < P) ++shift;
  const uint64_t max_keys = static_cast<uint64_t>(t->page_stride) << shift;
  *out = PagedKV{t->row_offsets, t->column_lengths, t->page_table, rows, columns / P, shift, t->page_stride,
                 static_cast<uint32_t>(max_keys < 0x7fffffffu ? max_keys : 0x7fffffffu), 0, t->count, t->max_row};
  return MFA_SUCCESS;
}

// The launch form of a paged K/V append (table and new tokens), after every check mfa_paged_kv_append makes before it
// looks for a device
static int append_of(const mfa_paged_kv_t *paged, const mfa_paged_kv_append_t *append, const void *k_pool,
                     const void *v_pool, PagedKV *pk, AppendSource *src) {
  if (!paged) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL paged K/V table.");
  if (!append) return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V append: NULL append.");
  const mfa_paged_kv_append_t &a = *append;
  if (!a.k_new || !a.v_new || !k_pool || !v_pool)
    return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Paged K/V append: ") +
                                                (!a.k_new ? "k_new" : !a.v_new ? "v_new" : !k_pool ? "k_pool" : "v_pool") +
                                                " must not be NULL.");
  const int status = paged_table_of(paged, a.rows, a.pool_rows, "rows", "pool_rows", pk);
  if (status != MFA_SUCCESS) return status;
  if (a.kv_heads == 0) return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V append: kv_heads 0 must be at least 1.");
  if (a.head_dimension == 0 || a.head_dimension > 512)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V append: head_dimension " + std::to_string(a.head_dimension) +
                                                " is outside [1, 512].");
  const uint64_t row_elements = static_cast<uint64_t>(a.kv_heads) * a.head_dimension;
  if (a.token_stride != 0 && a.token_stride < row_elements)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V append: token_stride " + std::to_string(a.token_stride) +
                                                " is below kv_heads * head_dimension = " + std::to_string(row_elements) +
                                                ".");
  if (row_elements > 0xffffffffu)  // (only reachable with token_stride 0: a nonzero stride bounds it)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V append: kv_heads * head_dimension = " +
                                                std::to_string(row_elements) + " exceeds 2^32 - 1.");
  if (a.precision > MFA_BF16)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V append: precision " + std::to_string(a.precision) +
                                                " is not MFA_FP32, MFA_FP16 or MFA_BF16.");
  pk->kv_heads = a.kv_heads;
  *src = AppendSource{a.k_new, a.v_new,
                      a.token_stride ? a.token_stride : static_cast<uint32_t>(row_elements), a.head_dimension,
                      static_cast<uint32_t>(row_elements), static_cast<uint8_t>(a.precision)};
  return MFA_SUCCESS;
}

// The launch form of a paged K/V table, after the checks the host can make without reading device memory
static int paged_of(const mfa_attention_kernel *k, const mfa_function_constants_t *c, const mfa_paged_kv_t *t,
                    PagedKV *out) {
  if (!t) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL paged K/V table.");
  if (k->type != MFA_FORWARD)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V: only the forward kernel reads a paged cache.");
  int n = 0;
  const int *ops = operands_of(k->type, &n);
  for (int i = 0; i < n; ++i)
    if ((k->descriptor.transpose_state_mask >> ops[i]) & 1)
      return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Paged K/V needs row-major operands; ") +
                                                  mfa_operand_name((mfa_operand_t)ops[i]) + " is transposed.");
  if (k->backend == MFA_BACKEND_TCGEN05 && k->descriptor.head_dimension % 8 != 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V on MFA_BACKEND_TCGEN05 needs a head dimension that is a multiple "
                                            "of 8 (head " + std::to_string(k->descriptor.head_dimension) + ").");
  int status = paged_table_of(t, c->row, c->column, "row", "column", out);
  if (status != MFA_SUCCESS) return status;
  const uint32_t batch = c->batch_count ? c->batch_count : 1;
  if (batch > kMaxBatchPerLaunch)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Paged K/V: batch_count " + std::to_string(batch) + " exceeds " +
                                                std::to_string(kMaxBatchPerLaunch) + " (a paged call is one launch).");
  uint32_t group = 1;
  if ((status = kv_group_of(c, &group)) != MFA_SUCCESS) return status;
  out->kv_heads = batch / group;
  return MFA_SUCCESS;
}

// A split-KV request (mfa_split_kv_t) of a call over call->seq or call->pk, after the checks the host can make; the
// table's checks come first.  The key bound the plan cuts is the hint, or the table's bound (capped so that block counts
// cannot overflow).
constexpr uint32_t kMaxKeySplits = 16;
static int split_of(const mfa_attention_kernel *k, const mfa_split_kv_t *s, AttentionCall *call) {
  if (!s) return fail(MFA_ERROR_INVALID_ARGUMENT, "Split-KV: NULL split.");
  if (k->type != MFA_FORWARD)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Split-KV: only the forward kernel splits its key range.");
  if (s->num_splits > kMaxKeySplits)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Split-KV: num_splits " + std::to_string(s->num_splits) + " is above " +
                                                std::to_string(kMaxKeySplits) + ".");
  const uint32_t bound = s->max_column ? s->max_column : (call->seq ? call->seq->max_column : call->pk->max_keys);
  call->split = true;
  call->num_splits = s->num_splits;
  call->key_bound = bound < 0x7fffffffu ? bound : 0x7fffffffu;
  return MFA_SUCCESS;
}
// An FP8 K/V request (mfa_fp8_kv_t), after the checks the host can make; the table's and the split's checks come first
// (paged_of rejects every kernel but the forward)
static int fp8_of(const mfa_attention_kernel *k, const mfa_fp8_kv_t *f, Fp8KV *out) {
  if (!f) return fail(MFA_ERROR_INVALID_ARGUMENT, "FP8 K/V: NULL fp8.");
  if (k->backend != MFA_BACKEND_TCGEN05)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "FP8 K/V needs the tensor-core family (MFA_BACKEND_TCGEN05); this kernel "
                                            "is on MFA_BACKEND_SIMT_FP32.");
  if (k->descriptor.head_dimension % 16 != 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "FP8 K/V needs a head dimension that is a multiple of 16 (head " +
                                                std::to_string(k->descriptor.head_dimension) +
                                                "): TMA reads the pools' 1-byte rows at 16-byte strides.");
  *out = Fp8KV{f->k_scale, f->v_scale};
  return MFA_SUCCESS;
}

// The plan of a call on the tensor cores, per batch slice (a paged call is one slice), with the kernel's window:
// f(first problem of the slice, plan)
template <class F>
static int wgmma_plans(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c, AttentionCall call,
                       F f) {
  const mfa_attention_kernel_descriptor_t &d = kernel->descriptor;
  uint32_t group = 1;
  const int status = kv_group_of(c, &group);
  if (status != MFA_SUCCESS) return status;
  Band band;
  call.band = band_of(kernel, c->row, call.pk ? call.pk->max_keys : c->column, &band);
  const uint32_t Dp = (d.head_dimension + 7u) / 8u * 8u, sm_count = device_sm_count(current_device());
  // (only the dK/dV plan reads it)
  const bool convert_dO = d.memory_precisions[MFA_dO] != d.memory_precisions[MFA_Q];
  return for_each_batch_slice(c->batch_count ? c->batch_count : 1, group, [&](uint32_t h0, uint32_t batch) -> int {
    f(h0, wgmma_plan(kernel->type, Dp, c->row, c->column, batch, group, d.split_min_blocks,
                     d.split_max ? d.split_max : 1, convert_dO, call, sm_count));
    return MFA_SUCCESS;
  });
}

// The first checks of an encode over a sequence table or a paged cache, before the table's
static int encode_arguments(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *constants,
                            void *const buffers[MFA_BUFFER_COUNT]) {
  if (!kernel || !constants || !buffers) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if (constants->row == 0 || constants->column == 0) return fail(MFA_ERROR_INVALID_ARGUMENT, "R and C must be at least 1.");
  return MFA_SUCCESS;
}

// encode() of any kernel type in the form `call` describes; the kernel's window is added to the call here
static int encode(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *constants, AttentionCall call,
                  void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream);

}  // namespace mfa

using namespace mfa;

extern "C" {

int mfa_attention_kernel_create(const mfa_attention_kernel_descriptor_t *kd, mfa_attention_kernel_t **out) {
  if (!kd || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  // guard let ... else fatalError("Descriptor was incomplete.")  (AttentionKernel.swift:28-34)
  if (!kd->has_block_dimensions || !kd->has_head_dimension || kd->prefer_async_cache == 0xFF ||
      kd->prefer_async_load == 0xFF || kd->type == 0xFF)
    return fail(MFA_ERROR_INCOMPLETE_DESCRIPTOR, "Descriptor was incomplete.");
  if (kd->type > MFA_BACKWARD_KEY_VALUE) return fail(MFA_ERROR_INVALID_ARGUMENT, "Unrecognized kernel type.");
  if (kd->head_dimension == 0) return fail(MFA_ERROR_INVALID_ARGUMENT, "Head dimension must be at least 1.");
  if (kd->causal > 1) return fail(MFA_ERROR_INVALID_ARGUMENT, "Unrecognized causal mask mode.");

  int n = 0;
  const int *ops = operands_of(kd->type, &n);
  for (int i = 0; i < n; ++i) {
    int op = ops[i];
    uint8_t mem = kd->memory_precisions[op], reg = kd->register_precisions[op];
    if (mem == 0xFF || reg == 0xFF)
      return fail(MFA_ERROR_INCOMPLETE_DESCRIPTOR,
                  std::string("Precision of ") + mfa_operand_name((mfa_operand_t)op) + " was not specified.");
    if (!precision_pair_valid(mem, reg)) return fail(MFA_ERROR_INVALID_PRECISIONS, "Invalid precisions.");
    if (op != MFA_L && op != MFA_D && !((kd->transpose_state_valid_mask >> op) & 1))
      return fail(MFA_ERROR_INCOMPLETE_DESCRIPTOR,
                  std::string("Transpose state of ") + mfa_operand_name((mfa_operand_t)op) + " was not specified.");
  }

  mfa_attention_kernel *k = new mfa_attention_kernel();
  k->descriptor = *kd;
  k->type = kd->type;
  k->backend = kd->backend;
  const uint32_t D = kd->head_dimension;

  if (k->backend == MFA_BACKEND_TCGEN05) {
    // The tensor-core kernels only exist for 16-bit row-major operands; reject descriptors edited into
    // something they cannot serve instead of silently computing something else.
    const uint8_t pq = kd->memory_precisions[MFA_Q];
    const uint32_t Dp = (D + 7) / 8 * 8;  // D % 8 != 0: operands are staged with pad8(D) columns (kernels/pad_head.cu)
    bool ok = (pq == MFA_FP16 || pq == MFA_BF16) && kd->memory_precisions[MFA_K] == pq &&
              kd->memory_precisions[MFA_V] == pq && Dp <= kWgmmaMaxHead;
    bool transposed = false;
    for (int i = 0; i < n; ++i)
      if ((kd->transpose_state_mask >> ops[i]) & 1) transposed = true;
    if (transposed && D % 8 != 0) ok = false;  // padding is implemented for row-major operands
    // dO: same element type, or BF16 beside FP16 Q/K/V (the reference's policy; converted on chip)
    if (k->type != MFA_FORWARD && kd->memory_precisions[MFA_dO] != pq &&
        !(pq == MFA_FP16 && kd->memory_precisions[MFA_dO] == MFA_BF16))
      ok = false;
    if (!ok) {
      delete k;
      return fail(MFA_ERROR_UNSUPPORTED,
                  "MFA_BACKEND_TCGEN05 needs FP16/BF16 Q,K,V (row-major for head % 8 != 0; dO of the same "
                  "type, or BF16 with FP16 Q,K,V) and pad8(head) <= the compiled maximum; use MFA_BACKEND_SIMT_FP32 for this "
                  "descriptor.");
    }
    // (only the geometry fields are used: they depend on neither the problem size nor the device)
    const WgmmaPlan plan = wgmma_plan(k->type, Dp, 1, 1, 1, 1, 0, 1, false, AttentionCall{}, 1);
    k->threads = plan.threads;
    k->smem_bytes = plan.smem_bytes;
    k->par = plan.par;
    k->trav = plan.trav;
    k->head = plan.head;
  } else if (k->backend == MFA_BACKEND_SIMT_FP32) {
    if (D > 512) {
      delete k;
      return fail(MFA_ERROR_UNSUPPORTED, "Head dimension " + std::to_string(D) + " exceeds 512.");
    }
    simt_geometry(k->type, D, &k->threads, &k->smem_bytes, &k->par, &k->trav, &k->head);
  } else {
    delete k;
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Unrecognized backend.");
  }
  // The kernel object reports the tile shape the compiled kernel really uses; a descriptor whose
  // block dimensions were edited away from a compiled configuration is rejected.
  if (kd->block_parallelization != k->par || kd->block_traversal != k->trav) {
    std::string msg = "Block dimensions " + std::to_string(kd->block_parallelization) + "x" +
                      std::to_string(kd->block_traversal) + " have no compiled sm_90a kernel (available: " +
                      std::to_string(k->par) + "x" + std::to_string(k->trav) + ").";
    delete k;
    return fail(MFA_ERROR_UNSUPPORTED, msg);
  }
  static const char *typeNames[] = {"forward", "backward_query", "backward_key_value"};
  k->source_name = std::string("attention_") + typeNames[k->type] +
                   (k->backend == MFA_BACKEND_TCGEN05 ? "_tcgen05" : "_simt_fp32") + "<D=" + std::to_string(D) +
                   ">" + (kd->causal ? "_causal" : "");
  k->windowed = false;
  k->window = mfa_attention_window_t{-1, -1};
  *out = k;
  return MFA_SUCCESS;
}

int mfa_attention_kernel_create_windowed(const mfa_attention_kernel_descriptor_t *kd, const mfa_attention_window_t *window,
                                         mfa_attention_kernel_t **out) {
  if (!kd || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if (!window) return fail(MFA_ERROR_INVALID_ARGUMENT, "Window: NULL window.");
  if (window->left < -1)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Window: left " + std::to_string(window->left) + " is below -1.");
  if (window->right < -1)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Window: right " + std::to_string(window->right) + " is below -1.");
  if (kd->causal && window->right > 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Window: right " + std::to_string(window->right) +
                                                " on a causal kernel, whose band ends at the diagonal (0 or -1).");
  mfa_attention_kernel_t *k = nullptr;
  const int status = mfa_attention_kernel_create(kd, &k);
  if (status != MFA_SUCCESS) return status;
  k->windowed = true;
  k->window = *window;
  k->source_name += "_window<" + std::to_string(window->left) + "," + std::to_string(window->right) + ">";
  *out = k;
  return MFA_SUCCESS;
}

void mfa_attention_kernel_destroy(mfa_attention_kernel_t *kernel) { delete kernel; }

int mfa_attention_kernel_block_dimensions(const mfa_attention_kernel_t *kernel, uint16_t out[3]) {
  if (!kernel || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  out[0] = static_cast<uint16_t>(kernel->par);
  out[1] = static_cast<uint16_t>(kernel->trav);
  out[2] = static_cast<uint16_t>(kernel->head);
  return MFA_SUCCESS;
}

int mfa_attention_kernel_threadgroup_size(const mfa_attention_kernel_t *kernel, uint32_t *out) {
  if (!kernel || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  *out = kernel->threads;
  return MFA_SUCCESS;
}

int mfa_attention_kernel_threadgroup_memory_allocation(const mfa_attention_kernel_t *kernel, uint32_t *out) {
  if (!kernel || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  *out = kernel->smem_bytes;
  return MFA_SUCCESS;
}

namespace mfa {
static int grid_size(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                     const AttentionCall &call, uint32_t *out) {
  if (kernel->backend == MFA_BACKEND_TCGEN05) {
    *out = 0;  // the CTAs of one traversal range
    return wgmma_plans(kernel, c, call, [&](uint32_t, const WgmmaPlan &plan) {
      *out += static_cast<uint32_t>(static_cast<uint64_t>(plan.grid.x) * plan.grid.y * plan.grid.z / plan.splits);
    });
  }
  // parallelization dimension: R for forward / backwardQuery, C for backwardKeyValue
  // (AttentionKernel.swift:197-204; dispatch: SquareAttentionTest.swift:328-339)
  // (dK/dV: one CTA per K/V tile, which walks the query problems of its group; packed sequences and paged calls: the
  // tiles of the longest sequence, once per sequence)
  const bool key_value = kernel->type == MFA_BACKWARD_KEY_VALUE;
  const Sequences *seq = call.seq;
  const uint32_t dim = call.pk ? call.pk->max_row
                               : (key_value ? (seq ? seq->max_column : c->column) : (seq ? seq->max_row : c->row));
  const uint32_t count = call.pk ? call.pk->count : (seq ? seq->count : 1);
  const uint32_t batch = c->batch_count ? c->batch_count : 1;
  uint32_t group = 1;
  const int status = kv_group_of(c, &group);
  if (status != MFA_SUCCESS) return status;
  *out = ((dim + kernel->par - 1) / kernel->par) * (key_value ? batch / group : batch) * count;
  return MFA_SUCCESS;
}

static int launch_count(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                        const AttentionCall &call, uint32_t *out) {
  *out = 0;
  if (kernel->backend == MFA_BACKEND_TCGEN05) {
    const uint32_t staged = __builtin_popcount(staged_operands(kernel));
    return wgmma_plans(kernel, c, call, [&](uint32_t, const WgmmaPlan &plan) { *out += staged + plan.launches; });
  }
  uint32_t group = 1;
  const int status = kv_group_of(c, &group);
  if (status != MFA_SUCCESS) return status;
  return for_each_batch_slice(c->batch_count ? c->batch_count : 1, group, [&](uint32_t, uint32_t) -> int {
    *out += 1;
    return MFA_SUCCESS;
  });
}

// The plan of a split-KV call: the forward plan's on the tensor cores, one split on the SIMT family
static int split_plan(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                      const AttentionCall &call, mfa_split_plan_t *out) {
  *out = mfa_split_plan_t{1, 1, 0, 0};
  if (kernel->backend != MFA_BACKEND_TCGEN05) {
    const int status = grid_size(kernel, c, call, &out->grid_size);
    return status != MFA_SUCCESS ? status : launch_count(kernel, c, call, &out->launch_count);
  }
  const uint32_t staged = __builtin_popcount(staged_operands(kernel));
  return wgmma_plans(kernel, c, call, [&](uint32_t h0, const WgmmaPlan &plan) {
    if (h0 == 0) {
      out->splits = plan.splits;
      out->heads_per_tile = plan.heads_per_tile;
    }
    out->grid_size += plan.grid.x * plan.grid.y * plan.grid.z;
    out->launch_count += staged + plan.launches;
  });
}
}  // namespace mfa

int mfa_attention_kernel_grid_size(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                   uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  return grid_size(kernel, c, AttentionCall{}, out);
}

int mfa_attention_kernel_grid_size_sequences(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                             const mfa_sequence_table_t *table, uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  Sequences seq;
  AttentionCall call{&seq};
  const int status = sequences_of(kernel, c, table, &seq);
  return status != MFA_SUCCESS ? status : grid_size(kernel, c, call, out);
}

const char *mfa_attention_kernel_source_name(const mfa_attention_kernel_t *kernel) {
  return kernel ? kernel->source_name.c_str() : "";
}

int mfa_attention_kernel_launch_count(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                      uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  return launch_count(kernel, c, AttentionCall{}, out);
}

int mfa_attention_kernel_launch_count_sequences(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                                const mfa_sequence_table_t *table, uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  Sequences seq;
  AttentionCall call{&seq};
  const int status = sequences_of(kernel, c, table, &seq);
  return status != MFA_SUCCESS ? status : launch_count(kernel, c, call, out);
}

int mfa_attention_kernel_encode(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *constants,
                                void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream) {
  if (!kernel || !constants || !buffers) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  return encode(kernel, constants, AttentionCall{}, buffers, cuda_stream);
}

int mfa_attention_kernel_grid_size_paged(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                         const mfa_paged_kv_t *table, uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  PagedKV pk;
  AttentionCall call{nullptr, &pk};
  const int status = paged_of(kernel, c, table, &pk);
  return status != MFA_SUCCESS ? status : grid_size(kernel, c, call, out);
}

int mfa_attention_kernel_launch_count_paged(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                            const mfa_paged_kv_t *table, uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  PagedKV pk;
  AttentionCall call{nullptr, &pk};
  const int status = paged_of(kernel, c, table, &pk);
  return status != MFA_SUCCESS ? status : launch_count(kernel, c, call, out);
}

int mfa_attention_kernel_split_plan(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                    const mfa_sequence_table_t *sequences, const mfa_paged_kv_t *paged,
                                    const mfa_split_kv_t *split, mfa_split_plan_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if ((sequences != nullptr) == (paged != nullptr))
    return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Split-KV: pass exactly one of sequences and paged (") +
                                                (sequences ? "both" : "neither") + " given).");
  Sequences seq;
  PagedKV pk;
  AttentionCall call{sequences ? &seq : nullptr, paged ? &pk : nullptr};
  int status = sequences ? sequences_of(kernel, c, sequences, &seq) : paged_of(kernel, c, paged, &pk);
  if (status != MFA_SUCCESS || (status = split_of(kernel, split, &call)) != MFA_SUCCESS) return status;
  return split_plan(kernel, c, call, out);
}

int mfa_attention_kernel_encode_paged(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *constants,
                                      const mfa_paged_kv_t *table, void *const buffers[MFA_BUFFER_COUNT],
                                      void *cuda_stream) {
  PagedKV pk;
  AttentionCall call{nullptr, &pk};
  int status = encode_arguments(kernel, constants, buffers);
  if (status != MFA_SUCCESS || (status = paged_of(kernel, constants, table, &pk)) != MFA_SUCCESS) return status;
  return encode(kernel, constants, call, buffers, cuda_stream);
}

int mfa_attention_kernel_encode_sequences(const mfa_attention_kernel_t *kernel,
                                          const mfa_function_constants_t *constants, const mfa_sequence_table_t *table,
                                          void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream) {
  Sequences seq;
  AttentionCall call{&seq};
  int status = encode_arguments(kernel, constants, buffers);
  if (status != MFA_SUCCESS || (status = sequences_of(kernel, constants, table, &seq)) != MFA_SUCCESS) return status;
  return encode(kernel, constants, call, buffers, cuda_stream);
}

int mfa_attention_kernel_encode_paged_split(const mfa_attention_kernel_t *kernel,
                                            const mfa_function_constants_t *constants, const mfa_paged_kv_t *table,
                                            const mfa_split_kv_t *split, void *const buffers[MFA_BUFFER_COUNT],
                                            void *cuda_stream) {
  PagedKV pk;
  AttentionCall call{nullptr, &pk};
  int status = encode_arguments(kernel, constants, buffers);
  if (status != MFA_SUCCESS || (status = paged_of(kernel, constants, table, &pk)) != MFA_SUCCESS ||
      (status = split_of(kernel, split, &call)) != MFA_SUCCESS)
    return status;
  return encode(kernel, constants, call, buffers, cuda_stream);
}

int mfa_attention_kernel_encode_paged_fp8(const mfa_attention_kernel_t *kernel,
                                          const mfa_function_constants_t *constants, const mfa_paged_kv_t *table,
                                          const mfa_split_kv_t *split, const mfa_fp8_kv_t *fp8,
                                          void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream) {
  PagedKV pk;
  Fp8KV scales;
  AttentionCall call{nullptr, &pk, nullptr, &scales};
  int status = encode_arguments(kernel, constants, buffers);
  if (status != MFA_SUCCESS || (status = paged_of(kernel, constants, table, &pk)) != MFA_SUCCESS ||
      (split && (status = split_of(kernel, split, &call)) != MFA_SUCCESS) ||
      (status = fp8_of(kernel, fp8, &scales)) != MFA_SUCCESS)
    return status;
  return encode(kernel, constants, call, buffers, cuda_stream);
}

int mfa_attention_kernel_encode_sequences_split(const mfa_attention_kernel_t *kernel,
                                                const mfa_function_constants_t *constants,
                                                const mfa_sequence_table_t *table, const mfa_split_kv_t *split,
                                                void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream) {
  Sequences seq;
  AttentionCall call{&seq};
  int status = encode_arguments(kernel, constants, buffers);
  if (status != MFA_SUCCESS || (status = sequences_of(kernel, constants, table, &seq)) != MFA_SUCCESS ||
      (status = split_of(kernel, split, &call)) != MFA_SUCCESS)
    return status;
  return encode(kernel, constants, call, buffers, cuda_stream);
}

int mfa_paged_kv_append(const mfa_paged_kv_t *paged, const mfa_paged_kv_append_t *append, void *k_pool, void *v_pool,
                        const mfa_fp8_kv_t *fp8, void *cuda_stream) {
  PagedKV pk;
  AppendSource src;
  int status = append_of(paged, append, k_pool, v_pool, &pk, &src);
  if (status != MFA_SUCCESS || (status = check_device()) != MFA_SUCCESS) return status;
  Fp8KV scales{};
  if (fp8) scales = Fp8KV{fp8->k_scale, fp8->v_scale};
  const cudaError_t e = launch_paged_kv_append(pk, src, k_pool, v_pool, fp8 ? &scales : nullptr,
                                               static_cast<cudaStream_t>(cuda_stream));
  if (e != cudaSuccess)
    return fail(MFA_ERROR_CUDA, std::string("launch of paged_kv_append failed: ") + cudaGetErrorString(e));
  return MFA_SUCCESS;
}

int mfa_paged_kv_append_rotary(const mfa_paged_kv_t *paged, const mfa_paged_kv_append_t *append,
                               const mfa_rotary_t *rotary, void *k_pool, void *v_pool, const mfa_fp8_kv_t *fp8,
                               void *cuda_stream) {
  PagedKV pk;
  AppendSource src;
  int status = append_of(paged, append, k_pool, v_pool, &pk, &src);
  if (status != MFA_SUCCESS) return status;
  if (!rotary) return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: NULL rotary.");
  const mfa_rotary_t &r = *rotary;
  if (!r.q_new || !r.q_out || !r.cos || !r.sin)
    return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Rotary append: ") +
                                                (!r.q_new ? "q_new" : !r.q_out ? "q_out" : !r.cos ? "cos" : "sin") +
                                                " must not be NULL.");
  if (r.query_heads == 0 || r.query_heads % pk.kv_heads != 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: query_heads " + std::to_string(r.query_heads) +
                                                " is not a positive multiple of kv_heads = " +
                                                std::to_string(pk.kv_heads) + ".");
  const uint64_t q_elements = static_cast<uint64_t>(r.query_heads) * src.head_dimension;
  if (q_elements > 0xffffffffu)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: query_heads * head_dimension = " +
                                                std::to_string(q_elements) + " exceeds 2^32 - 1.");
  if (r.q_token_stride != 0 && r.q_token_stride < q_elements)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: q_token_stride " + std::to_string(r.q_token_stride) +
                                                " is below query_heads * head_dimension = " +
                                                std::to_string(q_elements) + ".");
  if (r.rotary_dim == 0 || r.rotary_dim % 2 != 0 || r.rotary_dim > src.head_dimension)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: rotary_dim " + std::to_string(r.rotary_dim) +
                                                " must be even and in [2, head_dimension = " +
                                                std::to_string(src.head_dimension) + "].");
  if (r.table_stride != 0 && r.table_stride < r.rotary_dim / 2)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: table_stride " + std::to_string(r.table_stride) +
                                                " is below rotary_dim / 2 = " + std::to_string(r.rotary_dim / 2) + ".");
  const uint64_t keys = static_cast<uint64_t>(paged->page_stride) * paged->page_size;
  if (r.positions < keys)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: positions " + std::to_string(r.positions) +
                                                " is below page_stride * page_size = " + std::to_string(keys) + ".");
  if (r.interleaved > 1)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Rotary append: interleaved " + std::to_string(r.interleaved) +
                                                " is not 0 or 1.");
  if ((status = check_device()) != MFA_SUCCESS) return status;
  const RotarySource rot{r.q_new, r.q_out, r.cos, r.sin, r.query_heads,
                         r.q_token_stride ? r.q_token_stride : static_cast<uint32_t>(q_elements), r.rotary_dim,
                         r.table_stride ? r.table_stride : r.rotary_dim / 2, r.interleaved != 0};
  Fp8KV scales{};
  if (fp8) scales = Fp8KV{fp8->k_scale, fp8->v_scale};
  const cudaError_t e = launch_rotary_kv_append(pk, src, rot, k_pool, v_pool, fp8 ? &scales : nullptr,
                                                static_cast<cudaStream_t>(cuda_stream));
  if (e != cudaSuccess)
    return fail(MFA_ERROR_CUDA, std::string("launch of rotary_kv_append failed: ") + cudaGetErrorString(e));
  return MFA_SUCCESS;
}

}  // extern "C"

namespace mfa {
static int encode(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *constants, AttentionCall call,
                  void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream) {
  int status = check_device();
  if (status != MFA_SUCCESS) return status;
  AttentionParams p;
  status = build_params(kernel, constants, buffers, p);
  if (status != MFA_SUCCESS) return status;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  // (a paged call's keys are bounded by its table)
  Band storage;
  call.band = band_of(kernel, p.R, call.pk ? call.pk->max_keys : p.C, &storage);
  const Sequences *seq = call.seq;

  // Tensor-core family: operands with D % 8 != 0 or a transposed layout are staged row-major with pad8(D) columns, the
  // kernels run at the padded head dimension (the softmax scale stays 1 / sqrt(D) of the true D), and the FP32 outputs
  // are copied back to the caller's layout without the padding.
  size_t head_bytes[kSlots];
  for (int slot = 0; slot < kSlots; ++slot) {
    const size_t seq = key_value_slot(slot) ? p.C : p.R;
    const size_t elements = (slot == sL || slot == sD) ? seq : seq * p.D;
    head_bytes[slot] = elements * (p.prec[slot] == FP32 ? 4 : 2);
  }
  const uint32_t staged = staged_operands(kernel);
  const uint32_t Dp = (p.D + 7) / 8 * 8;
  const int device = staged ? current_device() : 0;
  auto seq_of = [&](int slot) -> uint32_t { return key_value_slot(slot) ? p.C : p.R; };
  return for_each_batch_slice(p.batch, p.group, [&](uint32_t h0, uint32_t batch) -> int {
    AttentionParams q = p;
    q.batch = batch;
    // the problems of a slot in this slice: K, V, dK and dV hold one per group
    auto problems_of = [&](int slot) -> uint32_t { return key_value_slot(slot) ? batch / p.group : batch; };
    for (int slot = 0; slot < kSlots; ++slot)
      if (q.buf[slot])
        q.buf[slot] = static_cast<char *>(q.buf[slot]) + head_bytes[slot] * (key_value_slot(slot) ? h0 / p.group : h0);
    cudaError_t e = cudaSuccess;
    void *user_out[kSlots] = {};  // staged outputs: where the caller's copies go
    if (staged) {
      auto bytes_of = [&](int slot) -> size_t {
        return ((static_cast<size_t>(problems_of(slot)) * seq_of(slot) * Dp * (p.prec[slot] == FP32 ? 4 : 2)) + 255) &
               ~size_t(255);
      };
      size_t total = 0;
      for (int slot = 0; slot < kSlots; ++slot)
        if ((staged >> slot) & 1) total += bytes_of(slot);
      void *ws = nullptr;
      if ((e = workspace_for(device, stream, total, &ws, /*slot=*/1)) != cudaSuccess)
        return fail(MFA_ERROR_CUDA, std::string("staging workspace: ") + cudaGetErrorString(e) + " " + last_launch_detail());
      char *cursor = static_cast<char *>(ws);
      for (int slot = 0; slot < kSlots && e == cudaSuccess; ++slot) {
        if (!((staged >> slot) & 1)) continue;
        if (is_output(kernel->type, slot))
          user_out[slot] = q.buf[slot];
        else
          e = launch_stage_operand(q.buf[slot], cursor, problems_of(slot), seq_of(slot), p.D, Dp,
                                   p.prec[slot] == FP32 ? 4 : 2, q.transposed[slot], stream);
        q.buf[slot] = cursor;
        cursor += bytes_of(slot);
      }
      for (int slot = 0; slot < kSlots; ++slot) q.transposed[slot] = 0;
      q.D = Dp;  // (q.scale / q.scale_log2 keep the true head dimension)
      if (e != cudaSuccess) return fail(MFA_ERROR_CUDA, std::string("operand staging failed: ") + cudaGetErrorString(e));
    }
    e = kernel->backend == MFA_BACKEND_TCGEN05 ? launch_wgmma(kernel->type, q, call, stream)
                                               : launch_simt(kernel->type, q, call, stream);
    if (e != cudaSuccess)
      return fail(MFA_ERROR_CUDA, std::string("launch of ") + kernel->source_name +
                                      (call.fp8 ? " (paged FP8 K/V)" : (call.pk ? " (paged K/V)" : "")) + " failed: " +
                                      cudaGetErrorString(e) + " " + last_launch_detail());
    // (packed sequences: only the sequences' rows, which the kernels wrote; the caller's other rows stay as they are)
    for (int slot = 0; slot < kSlots && e == cudaSuccess; ++slot)
      if (user_out[slot] && seq)
        e = launch_unstage_sequences(static_cast<const float *>(q.buf[slot]), static_cast<float *>(user_out[slot]),
                                     problems_of(slot), seq_of(slot),
                                     key_value_slot(slot) ? seq->column_offsets : seq->row_offsets, seq->count,
                                     key_value_slot(slot) ? seq->max_column : seq->max_row, p.D, Dp,
                                     p.transposed[slot], stream);
      else if (user_out[slot])
        e = launch_unstage_output(static_cast<const float *>(q.buf[slot]), static_cast<float *>(user_out[slot]),
                                  problems_of(slot), seq_of(slot), p.D, Dp, p.transposed[slot], stream);
    if (e != cudaSuccess) return fail(MFA_ERROR_CUDA, std::string("copy-back of staged outputs failed: ") + cudaGetErrorString(e));
    return MFA_SUCCESS;
  });
}
}  // namespace mfa

extern "C" {

// ------------------------------------------------------------------------------------------------
// Kernel cache keyed by descriptor -- the useful half of the reference's pipeline cache
// (GEMMKernel.pipelineCache / register(descriptor:), GEMM/GEMMDescriptor/GEMMDescriptor+PipelineCache.swift:16-36):
// the reference caches (kernel, MTLComputePipelineState) per problem descriptor because a Metal JIT compile costs
// milliseconds; here the kernels are compiled ahead of time, so what is worth keeping is the validated kernel object.
// Handles returned from the cache are owned by the library and live until process exit.
// ------------------------------------------------------------------------------------------------
namespace {
struct CacheKey {
  mfa_attention_descriptor_t descriptor;
  int type;
  unsigned table_generation;  // kernels created from an older parameter table are not handed out again
  bool windowed;
  mfa_attention_window_t window;
};
std::mutex g_cache_mutex;
std::vector<std::pair<CacheKey, mfa_attention_kernel_t *>> g_kernel_cache;

bool same_descriptor(const mfa_attention_descriptor_t &a, const mfa_attention_descriptor_t &b) {
  // field-wise (struct padding is not part of the value); the matrix dimensions R, C and the batch count are launch-time
  // constants (setFunctionConstants), not part of the kernel -- only the head dimension is
  return a.low_precision_inputs == b.low_precision_inputs &&
         a.low_precision_intermediates == b.low_precision_intermediates &&
         a.has_matrix_dimensions == b.has_matrix_dimensions && a.has_transpose_state == b.has_transpose_state &&
         a.head == b.head && a.transpose_Q == b.transpose_Q && a.transpose_K == b.transpose_K &&
         a.transpose_V == b.transpose_V && a.transpose_O == b.transpose_O &&
         a.input_precision_override == b.input_precision_override && a.causal == b.causal &&
         // with transposed operands the kernel family depends on R % 8 / C % 8 (TMA row pitch)
         select_backend(a, MFA_FORWARD) == select_backend(b, MFA_FORWARD);
}
}  // namespace

namespace {
// window: nullptr for a kernel without one
int cache_fetch(const mfa_attention_descriptor_t *descriptor, mfa_kernel_type_t type,
                const mfa_attention_window_t *window, const mfa_attention_kernel_t **out) {
  std::lock_guard<std::mutex> lock(g_cache_mutex);
  for (const auto &entry : g_kernel_cache)
    if (entry.first.type == static_cast<int>(type) && entry.first.table_generation == parameter_table_generation() &&
        entry.first.windowed == (window != nullptr) &&
        (!window || (entry.first.window.left == window->left && entry.first.window.right == window->right)) &&
        same_descriptor(entry.first.descriptor, *descriptor)) {
      *out = entry.second;
      return MFA_SUCCESS;
    }
  mfa_attention_kernel_descriptor_t kd;
  int status = mfa_attention_descriptor_kernel_descriptor(descriptor, type, &kd);
  if (status != MFA_SUCCESS) return status;
  mfa_attention_kernel_t *kernel = nullptr;
  if ((status = window ? mfa_attention_kernel_create_windowed(&kd, window, &kernel)
                       : mfa_attention_kernel_create(&kd, &kernel)) != MFA_SUCCESS)
    return status;
  g_kernel_cache.push_back({CacheKey{*descriptor, static_cast<int>(type), parameter_table_generation(), window != nullptr,
                                     window ? *window : mfa_attention_window_t{-1, -1}},
                            kernel});
  *out = kernel;
  return MFA_SUCCESS;
}
}  // namespace

int mfa_attention_kernel_cache_fetch(const mfa_attention_descriptor_t *descriptor, mfa_kernel_type_t type,
                                     const mfa_attention_kernel_t **out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  return cache_fetch(descriptor, type, nullptr, out);
}

int mfa_attention_kernel_cache_fetch_windowed(const mfa_attention_descriptor_t *descriptor, mfa_kernel_type_t type,
                                              const mfa_attention_window_t *window,
                                              const mfa_attention_kernel_t **out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if (!window) return fail(MFA_ERROR_INVALID_ARGUMENT, "Window: NULL window.");
  return cache_fetch(descriptor, type, window, out);
}

int mfa_attention_kernel_cache_size(void) {
  std::lock_guard<std::mutex> lock(g_cache_mutex);
  return static_cast<int>(g_kernel_cache.size());
}

// ------------------------------------------------------------------------------------------------
// Host-buffer path: H2D -> kernels -> D2H (the end-to-end call bench.py times as `e2e`).
//
// The independent single-head problems of a batch are cut into chunks that flow through three streams -- upload,
// compute, download -- linked by one event pair per chunk, so the host->device copy of chunk i+1, the kernels of chunk
// i and the device->host copy of chunk i-1 overlap (PCIe is full duplex and the GPU has a copy engine per direction) and
// the upload stream never waits for anything.  With pinned host buffers the call then costs max(H2D, D2H) + one chunk
// of fill/drain instead of H2D + kernels + D2H.
// ------------------------------------------------------------------------------------------------
namespace {
constexpr int kHostStreams = 3;  // 0 upload, 1 compute, 2 download
constexpr uint32_t kMaxChunks = 32;
struct Scratch {
  void *ptr[MFA_BUFFER_COUNT] = {};
  size_t bytes[MFA_BUFFER_COUNT] = {};
  bool ready = false;  // streams and events exist
  cudaStream_t stream[kHostStreams] = {};
  cudaEvent_t uploaded[kMaxChunks] = {}, computed[kMaxChunks] = {};
};
// One scratch set per (calling thread, device): a thread that alternates between devices keeps both sets, nothing
// leaks on a device switch, and a set is only marked ready once every stream and event exists.  Released by
// mfa_release_device_resources() (thread exit does not free device memory: the context may already be gone).
thread_local std::map<int, Scratch> g_scratch;

// RAII: mfa_attention_run_host selects `device` for the duration of the call and restores the caller's device
struct DeviceGuard {
  int previous = -1;
  bool active = false;
  cudaError_t enter(int device) {
    if (cudaGetDevice(&previous) != cudaSuccess) {
      cudaGetLastError();
      previous = -1;
    }
    cudaError_t e = cudaSetDevice(device);
    active = e == cudaSuccess && previous >= 0 && previous != device;
    return e;
  }
  ~DeviceGuard() {
    if (active) cudaSetDevice(previous);
  }
};

void destroy_scratch(Scratch &s) {
  for (int i = 0; i < MFA_BUFFER_COUNT; ++i) {
    if (s.ptr[i]) cudaFree(s.ptr[i]);
    s.ptr[i] = nullptr;
    s.bytes[i] = 0;
  }
  for (int i = 0; i < kHostStreams; ++i)
    if (s.stream[i]) cudaStreamDestroy(s.stream[i]);
  for (uint32_t i = 0; i < kMaxChunks; ++i) {
    if (s.uploaded[i]) cudaEventDestroy(s.uploaded[i]);
    if (s.computed[i]) cudaEventDestroy(s.computed[i]);
  }
  s = Scratch();
}

// heads per chunk: about sixteen chunks (fill + drain = two chunk times), but no chunk smaller than ~4 MB of traffic
// (copy launch overheads), at most kMaxChunks chunks, and no chunking at all for a single problem
uint32_t chunk_heads(uint32_t batch, size_t bytes_per_head) {
  if (batch <= 1) return 1;
  uint32_t heads = (batch + 15) / 16;
  const size_t kMinChunkBytes = size_t(4) << 20;
  if (bytes_per_head * heads < kMinChunkBytes)
    heads = static_cast<uint32_t>((kMinChunkBytes + bytes_per_head - 1) / bytes_per_head);
  if ((batch + heads - 1) / heads > kMaxChunks) heads = (batch + kMaxChunks - 1) / kMaxChunks;
  return heads < batch ? heads : batch;
}
}  // namespace

int mfa_attention_run_host(const mfa_attention_descriptor_t *descriptor, uint32_t run_mask,
                           void *const host_buffers[MFA_BUFFER_COUNT], int device) {
  if (!descriptor || !host_buffers) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if (!(run_mask & 7u)) return fail(MFA_ERROR_INVALID_ARGUMENT, "run_mask selects no kernel.");
  DeviceGuard guard;  // the caller's current device is restored on every exit
  cudaError_t e = guard.enter(device);
  if (e != cudaSuccess)
    return fail(MFA_ERROR_NO_DEVICE, std::string("cudaSetDevice: ") + cudaGetErrorString(e) +
                                         " (this library has no CPU fallback).");
  Scratch &s = g_scratch[device];
  if (!s.ready) {
    for (int i = 0; i < kHostStreams && e == cudaSuccess; ++i)
      e = cudaStreamCreateWithFlags(&s.stream[i], cudaStreamNonBlocking);
    for (uint32_t i = 0; i < kMaxChunks && e == cudaSuccess; ++i) {
      e = cudaEventCreateWithFlags(&s.uploaded[i], cudaEventDisableTiming);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.computed[i], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) {
      destroy_scratch(s);  // never leave a half-initialised set behind
      return fail(MFA_ERROR_CUDA, std::string("stream / event creation: ") + cudaGetErrorString(e));
    }
    s.ready = true;
  }

  // which operands each kernel reads / writes (AttentionKernelType.swift:10-22)
  uint32_t inputs = 0, outputs = 0;
  if (run_mask & MFA_RUN_FORWARD) {
    inputs |= (1u << MFA_Q) | (1u << MFA_K) | (1u << MFA_V);
    outputs |= (1u << MFA_O) | (1u << MFA_L);
  }
  if (run_mask & MFA_RUN_BACKWARD_QUERY) {
    inputs |= (1u << MFA_Q) | (1u << MFA_K) | (1u << MFA_V) | (1u << MFA_dO);
    if (!(run_mask & MFA_RUN_FORWARD)) inputs |= (1u << MFA_O) | (1u << MFA_L);
    outputs |= (1u << MFA_D) | (1u << MFA_dQ);
  }
  if (run_mask & MFA_RUN_BACKWARD_KEY_VALUE) {
    inputs |= (1u << MFA_Q) | (1u << MFA_K) | (1u << MFA_V) | (1u << MFA_dO);
    if (!(run_mask & MFA_RUN_FORWARD)) inputs |= (1u << MFA_L);
    if (!(run_mask & MFA_RUN_BACKWARD_QUERY)) inputs |= (1u << MFA_D);
    outputs |= (1u << MFA_dV) | (1u << MFA_dK);
  }

  mfa_function_constants_t constants;
  int status = mfa_attention_descriptor_set_function_constants(descriptor, &constants);
  if (status != MFA_SUCCESS) return status;
  const uint32_t batch = constants.batch_count ? constants.batch_count : 1;

  void *dev[MFA_BUFFER_COUNT] = {};
  size_t head_bytes[MFA_BUFFER_COUNT] = {};  // bytes of one single-head problem, per operand
  size_t traffic_per_head = 0;
  for (int op = 0; op < MFA_BUFFER_COUNT; ++op) {
    if (!((inputs | outputs) & (1u << op))) continue;
    size_t elements = 0;
    status = mfa_attention_descriptor_operand_elements(descriptor, (mfa_operand_t)op, &elements);
    if (status != MFA_SUCCESS) return status;
    const size_t nbytes = elements * (memory_precision(*descriptor, op) == MFA_FP32 ? 4 : 2);
    head_bytes[op] = nbytes / batch;
    if (s.bytes[op] < nbytes) {
      if (s.ptr[op]) cudaFree(s.ptr[op]);
      s.ptr[op] = nullptr;
      s.bytes[op] = 0;
      if ((e = cudaMalloc(&s.ptr[op], nbytes)) != cudaSuccess)
        return fail(MFA_ERROR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
      s.bytes[op] = nbytes;
    }
    dev[op] = s.ptr[op];
    if ((inputs & (1u << op)) && !host_buffers[op])
      return fail(MFA_ERROR_INVALID_ARGUMENT,
                  std::string("Host buffer ") + mfa_operand_name((mfa_operand_t)op) + " is NULL.");
    if ((inputs & (1u << op)) || host_buffers[op]) traffic_per_head += head_bytes[op];
  }

  // reference order: forward -> backwardQuery -> backwardKeyValue (SquareAttentionTest.swift:355-368)
  const mfa_attention_kernel_t *kernels[3] = {};
  for (int type = MFA_FORWARD; type <= MFA_BACKWARD_KEY_VALUE; ++type)
    if (run_mask & (1u << type))
      if ((status = mfa_attention_kernel_cache_fetch(descriptor, (mfa_kernel_type_t)type, &kernels[type])) != MFA_SUCCESS)
        return status;

  const uint32_t per_chunk = chunk_heads(batch, traffic_per_head);
  cudaStream_t upload = s.stream[0], compute = s.stream[1], download = s.stream[2];
  // every exit drains the three streams: the call is synchronous and the scratch is reused by the next one
  auto drained = [&](int result) {
    for (int i = 0; i < kHostStreams; ++i) cudaStreamSynchronize(s.stream[i]);
    return result;
  };
  // per-row statistics (L, D: a few KB per head) are not worth one copy per chunk: they come back in ONE copy after the
  // last chunk (the download stream is then behind every kernel)
  uint32_t small_outputs = 0;
  if (per_chunk < batch)
    for (int op = 0; op < MFA_BUFFER_COUNT; ++op)
      if ((outputs & (1u << op)) && host_buffers[op] && head_bytes[op] * batch <= (size_t(4) << 20)) small_outputs |= 1u << op;
  uint32_t chunk_index = 0;
  for (uint32_t h0 = 0; h0 < batch; h0 += per_chunk, ++chunk_index) {
    const uint32_t heads = batch - h0 < per_chunk ? batch - h0 : per_chunk;
    void *chunk_dev[MFA_BUFFER_COUNT] = {};
    for (int op = 0; op < MFA_BUFFER_COUNT; ++op) {
      if (!dev[op]) continue;
      chunk_dev[op] = static_cast<char *>(dev[op]) + head_bytes[op] * h0;
      if (inputs & (1u << op)) {
        const char *src = static_cast<const char *>(host_buffers[op]) + head_bytes[op] * h0;
        if ((e = cudaMemcpyAsync(chunk_dev[op], src, head_bytes[op] * heads, cudaMemcpyHostToDevice, upload)) != cudaSuccess)
          return drained(fail(MFA_ERROR_CUDA, std::string("H2D copy: ") + cudaGetErrorString(e)));
      }
    }
    if ((e = cudaEventRecord(s.uploaded[chunk_index], upload)) != cudaSuccess ||
        (e = cudaStreamWaitEvent(compute, s.uploaded[chunk_index], 0)) != cudaSuccess)
      return drained(fail(MFA_ERROR_CUDA, std::string("event: ") + cudaGetErrorString(e)));
    mfa_function_constants_t chunk_constants = constants;
    chunk_constants.batch_count = heads;
    for (int type = MFA_FORWARD; type <= MFA_BACKWARD_KEY_VALUE; ++type)
      if (kernels[type] &&
          (status = mfa_attention_kernel_encode(kernels[type], &chunk_constants, chunk_dev, compute)) != MFA_SUCCESS)
        return drained(status);
    if ((e = cudaEventRecord(s.computed[chunk_index], compute)) != cudaSuccess ||
        (e = cudaStreamWaitEvent(download, s.computed[chunk_index], 0)) != cudaSuccess)
      return drained(fail(MFA_ERROR_CUDA, std::string("event: ") + cudaGetErrorString(e)));
    for (int op = 0; op < MFA_BUFFER_COUNT; ++op) {
      if (!(outputs & (1u << op)) || !host_buffers[op] || (small_outputs & (1u << op))) continue;
      char *dst = static_cast<char *>(host_buffers[op]) + head_bytes[op] * h0;
      if ((e = cudaMemcpyAsync(dst, chunk_dev[op], head_bytes[op] * heads, cudaMemcpyDeviceToHost, download)) != cudaSuccess)
        return drained(fail(MFA_ERROR_CUDA, std::string("D2H copy: ") + cudaGetErrorString(e)));
    }
  }
  for (int op = 0; op < MFA_BUFFER_COUNT; ++op)
    if (small_outputs & (1u << op))
      if ((e = cudaMemcpyAsync(host_buffers[op], dev[op], head_bytes[op] * batch, cudaMemcpyDeviceToHost, download)) != cudaSuccess)
        return drained(fail(MFA_ERROR_CUDA, std::string("D2H copy: ") + cudaGetErrorString(e)));
  // (the device scratch is reused by the next call on this thread: every stream must have drained before returning,
  // which the synchronous contract of this entry point requires anyway)
  for (int i = 0; i < kHostStreams; ++i)
    if ((e = cudaStreamSynchronize(s.stream[i])) != cudaSuccess)
      return fail(MFA_ERROR_CUDA, std::string("kernel execution failed: ") + cudaGetErrorString(e));
  return MFA_SUCCESS;
}

int mfa_release_device_resources(int device) {
  DeviceGuard guard;
  cudaError_t e = guard.enter(device);
  if (e != cudaSuccess) return fail(MFA_ERROR_NO_DEVICE, std::string("cudaSetDevice: ") + cudaGetErrorString(e));
  if ((e = cudaDeviceSynchronize()) != cudaSuccess)
    return fail(MFA_ERROR_CUDA, std::string("cudaDeviceSynchronize: ") + cudaGetErrorString(e));
  auto it = g_scratch.find(device);
  if (it != g_scratch.end()) {
    destroy_scratch(it->second);
    g_scratch.erase(it);
  }
  release_workspaces(device);
  return MFA_SUCCESS;
}

}  // extern "C"
