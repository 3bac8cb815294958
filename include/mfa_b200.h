/*
 * mfa_b200.h -- C ABI of the H100-native FlashAttention hot path that stands in for
 * philipturner/metal-flash-attention's attention path.
 *
 * The reference's boundary is a set of Swift value types that *describe* a kernel and hand the
 * caller a Metal source string plus launch geometry; the caller compiles, binds ten buffers and
 * dispatches (Tests/FlashAttentionTests/Attention/SquareAttentionTest.swift:226-380).  This
 * header keeps that shape 1:1 (same names, same fields, same validation rules) and moves the
 * part the reference leaves to its caller -- compile + bind + dispatch -- behind
 * mfa_attention_kernel_encode(), because on H100 the kernels are pre-compiled sm_90a CUDA.
 *
 * Conventions
 *   - Plain C: pointers, sizes, enums with fixed raw values.  No torch / C++ types.
 *   - Every function returns MFA_SUCCESS (0) or a negative mfa_status_t; the message for the
 *     calling thread is available from mfa_last_error().  Where the reference calls
 *     fatalError() the ABI returns an error with the reference's message text (a C ABI must not
 *     abort its host); the Swift / C++ / Python mirrors turn that back into a trap/exception.
 *   - The library never owns caller buffers.  Device entry points take device pointers and a
 *     cudaStream_t (as void*) and are asynchronous on that stream.  The *_host entry point takes
 *     host pointers and performs H2D -> kernels -> D2H itself.
 *   - A kernel handle is immutable after creation and may be encoded concurrently from several
 *     threads / streams.
 *   - There is NO CPU fallback: if no sm_90 device / driver is present, encode fails loudly
 *     with MFA_ERROR_NO_DEVICE.
 *
 * Reference citations use R/ = the reference's Sources/FlashAttention/.
 */
#ifndef MFA_B200_H
#define MFA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define MFA_API __attribute__((visibility("default")))
#else
#define MFA_API
#endif

/* ------------------------------------------------------------------------------------------ */
/* Status                                                                                      */
/* ------------------------------------------------------------------------------------------ */
typedef enum mfa_status {
  MFA_SUCCESS = 0,
  MFA_ERROR_INCOMPLETE_DESCRIPTOR = -1, /* "Descriptor was incomplete."  R/Attention/AttentionDescriptor/AttentionDescriptor.swift:89-91, AttentionKernel.swift:28-34 */
  MFA_ERROR_INVALID_ARGUMENT = -2,      /* NULL pointer, enum out of range, operand without a buffer */
  MFA_ERROR_UNEXPECTED_OPERAND = -3,    /* "Unexpected operand: X"  AttentionDescriptor.swift:69-74 */
  MFA_ERROR_INVALID_PRECISIONS = -4,    /* "Invalid precisions."  AttentionKernel.swift:90-105 */
  MFA_ERROR_UNSUPPORTED = -5,           /* shape outside what the sm_90a kernels cover (e.g. head > 512) */
  MFA_ERROR_NO_DEVICE = -6,             /* no CUDA device / not sm_90 -- never falls back to a CPU path */
  MFA_ERROR_CUDA = -7                   /* a CUDA runtime / driver call failed; message has the detail */
} mfa_status_t;

/** Thread-local, NUL-terminated description of the last error on the calling thread. */
MFA_API const char *mfa_last_error(void);

/** Library version / build info ("mfa_b200 x.y sm_90a").  0.5 appended mfa_attention_kernel_descriptor_t.causal and
 *  mfa_function_constants_t.kv_group. */
MFA_API const char *mfa_version(void);

/* ------------------------------------------------------------------------------------------ */
/* Enumerations (raw values are part of the ABI)                                               */
/* ------------------------------------------------------------------------------------------ */

/** = GEMMOperandPrecision raw values.  R/GEMM/GEMMOperandPrecision.swift:33-37 */
typedef enum mfa_precision { MFA_FP32 = 0, MFA_FP16 = 1, MFA_BF16 = 2 } mfa_precision_t;

/** Size of one scalar in bytes.  GEMMOperandPrecision.size, R/GEMM/GEMMOperandPrecision.swift:51-60 */
MFA_API int mfa_precision_size(mfa_precision_t precision);
/** "float" / "half" / "bfloat".  GEMMOperandPrecision.name, :39-48 */
MFA_API const char *mfa_precision_name(mfa_precision_t precision);

/** = AttentionKernelType.  R/Attention/AttentionKernelType.swift:8-23 */
typedef enum mfa_kernel_type {
  MFA_FORWARD = 0,           /* computes O and L */
  MFA_BACKWARD_QUERY = 1,    /* computes D and dQ; depends on L */
  MFA_BACKWARD_KEY_VALUE = 2 /* computes dK and dV; depends on L and D */
} mfa_kernel_type_t;

/** = AttentionOperand.  Values 0..9 ARE the buffer bindings (AttentionOperand.bufferBinding,
 *  R/Attention/AttentionOperand.swift:52-71); S, P, dP, dS are never materialised (binding nil). */
typedef enum mfa_operand {
  MFA_Q = 0, MFA_K = 1, MFA_V = 2, MFA_O = 3,
  MFA_L = 4, MFA_D = 5,
  MFA_dO = 6, MFA_dV = 7, MFA_dK = 8, MFA_dQ = 9,
  MFA_S = 10, MFA_P = 11, MFA_dP = 12, MFA_dS = 13,
  MFA_OPERAND_COUNT = 14
} mfa_operand_t;
#define MFA_BUFFER_COUNT 10

/** "Q", "K", ..., "dQ".  AttentionOperand.description, AttentionOperand.swift:29-50 */
MFA_API const char *mfa_operand_name(mfa_operand_t operand);
/** Buffer slot 0..9, or -1 for S/P/dP/dS.  AttentionOperand.bufferBinding, :52-71 */
MFA_API int mfa_operand_buffer_binding(mfa_operand_t operand);

/* ------------------------------------------------------------------------------------------ */
/* AttentionDescriptor   (R/Attention/AttentionDescriptor/AttentionDescriptor.swift:10-27)     */
/* ------------------------------------------------------------------------------------------ */
typedef struct mfa_attention_descriptor {
  uint8_t low_precision_inputs;        /* lowPrecisionInputs (Q, K, V, dO)            :12 */
  uint8_t low_precision_intermediates; /* lowPrecisionIntermediates (S,P,L,D,dP,dS)   :15 */
  uint8_t has_matrix_dimensions;       /* Swift optional `matrixDimensions != nil`    :20 */
  uint8_t has_transpose_state;         /* Swift optional `transposeState != nil`      :22 */
  uint32_t row;                        /* matrixDimensions.row    (output sequence length R) */
  uint32_t column;                     /* matrixDimensions.column (input sequence length C)  */
  uint16_t head;                       /* matrixDimensions.head   (head dimension D)         */
  uint8_t transpose_Q, transpose_K, transpose_V, transpose_O; /* transposeState :22 */
  /* ---- library extensions; all-zero reproduces the reference exactly ---- */
  uint8_t input_precision_override;    /* 0: reference policy (Q,K,V FP16 and dO BF16 when lowPrecisionInputs,
                                          AttentionDescriptor+Precisions.swift:13-23);
                                          MFA_BF16 (2): Q,K,V,dO are all BF16 in memory (north_star asks for bf16);
                                          MFA_FP16 (1): Q,K,V,dO are all FP16.
                                          Only meaningful with low_precision_inputs.  All three variants run on the
                                          tensor-core kernels (with the reference policy the backward kernels rewrite
                                          the staged BF16 dO tiles as FP16 on chip: wgmma cannot mix
                                          FP16 and BF16 operands in one MMA). */
  uint8_t causal;                      /* 0: every query row sees every key (reference).  1: causal mask, aligned
                                          bottom-right: with delta = column - row (signed), query row i sees key j
                                          iff j <= i + delta.  row == column is the usual lower-triangular mask; with
                                          row < column the queries are the last `row` positions of a `column`-long
                                          sequence (chunked prefill, KV cache).  With row > column the rows
                                          i < row - column see no key: their O row is 0 and L = +inf, their D and dQ
                                          row are 0 and they add nothing to dK / dV (P = exp2(S - L) = 0).  The same
                                          mask applies to every problem of the batch.  Other values are rejected by
                                          kernelDescriptor(type:) with MFA_ERROR_INVALID_ARGUMENT. */
  uint32_t batch_count;                /* 0 or 1: single head (reference). N > 1: N independent
                                          single-head problems, each operand stored back to back
                                          (operand i of problem b starts at b * elements(i)). */
} mfa_attention_descriptor_t;

/** AttentionDescriptor.init(): all false / nil / zero. */
MFA_API void mfa_attention_descriptor_init(mfa_attention_descriptor_t *descriptor);

/** descriptor.memoryPrecisions[operand]   (AttentionDescriptor+Precisions.swift:10-146).
 *  Operands without a buffer (S,P,dP,dS) -> MFA_ERROR_INVALID_ARGUMENT. */
MFA_API int mfa_attention_descriptor_memory_precision(const mfa_attention_descriptor_t *descriptor,
                                                      mfa_operand_t operand, mfa_precision_t *out);
/** descriptor.registerPrecisions[operand] (AttentionDescriptor+Precisions.swift:149-215), i.e. the
 *  precision the operand has while it is an MMA operand / accumulator on chip. */
MFA_API int mfa_attention_descriptor_register_precision(const mfa_attention_descriptor_t *descriptor,
                                                        mfa_operand_t operand, mfa_precision_t *out);

/* ------------------------------------------------------------------------------------------ */
/* AttentionKernelDescriptor   (R/Attention/AttentionKernelDescriptor.swift:7-48)              */
/* ------------------------------------------------------------------------------------------ */
typedef enum mfa_backend {
  MFA_BACKEND_SIMT_FP32 = 0, /* CUDA-core FP32 FMA kernels: any R, C, D <= 512, any transposes/precisions */
  MFA_BACKEND_TCGEN05 = 1    /* TMA + wgmma kernels: 16-bit inputs, pad8(D) <= 256 for all three kernel types
                                (transposed operands too, with D % 8 == 0, where the transposed row pitch is a multiple
                                of 16 bytes) */
} mfa_backend_t;

typedef struct mfa_attention_kernel_descriptor {
  /* blockDimensions (parallelization, traversal, head)                               :8-9   */
  uint8_t has_block_dimensions;
  uint16_t block_parallelization, block_traversal, block_head;
  /* cacheState: bit i set <=> operand i is kept resident on chip for the whole traversal
     (registers on Apple GPUs; SMEM / registers on H100).                      :12    */
  uint16_t cache_state_valid_mask; /* which operands have an entry at all */
  uint16_t cache_state_mask;
  /* headDimension                                                                    :15    */
  uint8_t has_head_dimension;
  uint16_t head_dimension;
  /* memoryPrecisions / registerPrecisions; 0xFF = no entry                           :17,25 */
  uint8_t memory_precisions[MFA_OPERAND_COUNT];
  uint8_t register_precisions[MFA_OPERAND_COUNT];
  /* preferAsyncCache / preferAsyncLoad: 0 false, 1 true, 0xFF nil.  On H100 "async" means the
     TMA (cp.async.bulk.tensor) path; both are true for MFA_BACKEND_TCGEN05.          :20,23 */
  uint8_t prefer_async_cache, prefer_async_load;
  /* transposeState: bit i set <=> operand i is stored [D][seq] (leading dim = seq).   :27-42 */
  uint16_t transpose_state_valid_mask;
  uint16_t transpose_state_mask;
  /* type; 0xFF = nil                                                                 :44    */
  uint8_t type;
  /* ---- library extension: which sm_90a kernel family the heuristic picked ---- */
  uint8_t backend; /* mfa_backend_t */
  /* ---- library extension: the tuning columns of the parameter-table row (tensor-core family).  Like blockDimensions
     they are plain data the caller may edit before AttentionKernel(descriptor:). ---- */
  uint8_t split_min_blocks;  /* small grids: a traversal range handed to one CTA has at least this many traversal
                                blocks (blockDimensions.traversal rows each); 0 = never split */
  uint8_t split_max;         /* small grids: at most this many ranges per tile (forward <= 16, backward <= 8) */
  /* ---- library extension: the causal mask of mfa_attention_descriptor_t.causal (0 off, 1 bottom-right), copied by
     kernelDescriptor(type:); editable like the fields above.  Other values are rejected by AttentionKernel(descriptor:).
     Causal kernels visit only the blocks of the attention matrix that hold a visible (query, key) pair. ---- */
  uint8_t causal;
} mfa_attention_kernel_descriptor_t;

/** AttentionKernelDescriptor.init(): everything nil / empty. */
MFA_API void mfa_attention_kernel_descriptor_init(mfa_attention_kernel_descriptor_t *kernel_descriptor);

/** Element access to memory_precisions / register_precisions for host languages that import C arrays awkwardly (Swift
 *  sees them as 14-tuples): returns the precision raw value or -1 when unset; set with value < 0 to clear. */
MFA_API int mfa_attention_kernel_descriptor_get_precision(const mfa_attention_kernel_descriptor_t *kernel_descriptor,
                                                          mfa_operand_t operand, int register_file);
MFA_API void mfa_attention_kernel_descriptor_set_precision(mfa_attention_kernel_descriptor_t *kernel_descriptor,
                                                           mfa_operand_t operand, int register_file, int value);

/** descriptor.kernelDescriptor(type:)  (AttentionDescriptor.swift:33-130): looks up the H100
 *  parameter table for (type, precision class), picks the first row with head <= max head
 *  (AttentionDescriptor+Parameters.swift:41-66), clamps the head block to pad8(D) (:41-54),
 *  validates the cached-operand list (:56-86) and mirrors the transposes onto dO/dV/dK/dQ
 *  (:96-111).  Errors: MFA_ERROR_INCOMPLETE_DESCRIPTOR, MFA_ERROR_UNEXPECTED_OPERAND. */
MFA_API int mfa_attention_descriptor_kernel_descriptor(const mfa_attention_descriptor_t *descriptor,
                                                       mfa_kernel_type_t type,
                                                       mfa_attention_kernel_descriptor_t *out);

/** The parameter table text that kernelDescriptor(type:) would parse for this descriptor -- the analogue of
 *  AttentionDescriptor.parameterFile(type:) (AttentionDescriptor+Parameters.swift:13-39).  Rows are the reference's
 *  "| maxD | par | trav | head | cached |" with, for the tcgen05 family, two tuning columns appended:
 *  "| min blocks per split | max splits |".  The returned pointer stays valid until the table is replaced. */
MFA_API const char *mfa_attention_descriptor_parameter_file(const mfa_attention_descriptor_t *descriptor,
                                                            mfa_kernel_type_t type);

/** The tables are DATA: this replaces the tensor-core-family table of `type` (`transposed` != 0: the table used with transposed operands, i.e. of the
 *  layout-generic kernels) with `text` in the format above; NULL restores the built-in table.  The text is
 *  parsed and validated first (unknown operand names, malformed rows and rows without the two tuning columns are
 *  rejected and the current table stays).  Kernels fetched from the descriptor-keyed cache afterwards follow the new
 *  table.  At load time the library also reads the file named by the environment variable MFA_B200_PARAMETER_FILE
 *  (sections "[forward]", "[backwardQuery]", "[backwardKeyValue]", each also as "[....transposed]"; parameters/h100.txt is
 *  one).  Not thread-safe against concurrent kernelDescriptor() calls. */
MFA_API int mfa_set_parameter_table(mfa_kernel_type_t type, int transposed, const char *text);

/** descriptor.setFunctionConstants(_:)  (AttentionDescriptor.swift:139-148): the two launch-time
 *  constants R (index 0) and C (index 1), plus the batch and K/V-group extensions. */
typedef struct mfa_function_constants {
  uint32_t row;         /* R, function constant 0 */
  uint32_t column;      /* C, function constant 1 */
  uint32_t batch_count; /* extension; 0/1 = single head */
  uint32_t kv_group;    /* extension (appended in 0.5): grouped-query / multi-query attention.  The number of query
                           problems that share one K/V problem; 0 or 1 = every problem has its own K and V.  Query
                           problem b (Q, O, L, D, dO, dQ) reads K/V problem b / kv_group; the K, V, dK and dV buffers
                           hold batch_count / kv_group problems back to back, and dK / dV are the sums over the
                           kv_group query problems of a group.  For PyTorch [B, Hq, N, D] queries and [B, Hkv, N, D]
                           keys / values: batch_count = B * Hq, kv_group = Hq / Hkv (the head mapping of
                           scaled_dot_product_attention(enable_gqa=True)).  batch_count must be a multiple of kv_group
                           and kv_group at most 16384, else encode / grid_size / launch_count return
                           MFA_ERROR_INVALID_ARGUMENT.  set_function_constants writes 0 (the descriptor describes no
                           grouping): set it afterwards.  Not part of any kernel or of the kernel cache's key. */
} mfa_function_constants_t;
MFA_API int mfa_attention_descriptor_set_function_constants(const mfa_attention_descriptor_t *descriptor,
                                                            mfa_function_constants_t *constants);

/* ------------------------------------------------------------------------------------------ */
/* AttentionKernel   (R/Attention/AttentionKernel/AttentionKernel.swift:11-50, 268-363)        */
/* ------------------------------------------------------------------------------------------ */
typedef struct mfa_attention_kernel mfa_attention_kernel_t; /* opaque */

/** AttentionKernel(descriptor:)  (:27-50).  Incomplete descriptor -> MFA_ERROR_INCOMPLETE_DESCRIPTOR;
 *  illegal memory/register precision pairs (:81-139) -> MFA_ERROR_INVALID_PRECISIONS. */
MFA_API int mfa_attention_kernel_create(const mfa_attention_kernel_descriptor_t *kernel_descriptor,
                                        mfa_attention_kernel_t **out);
MFA_API void mfa_attention_kernel_destroy(mfa_attention_kernel_t *kernel);

/** kernel.blockDimensions  (:22): out[0..2] = parallelization, traversal, head. */
MFA_API int mfa_attention_kernel_block_dimensions(const mfa_attention_kernel_t *kernel, uint16_t out[3]);
/** kernel.threadgroupSize  (:268-270): threads per CTA of the selected sm_90a kernel. */
MFA_API int mfa_attention_kernel_threadgroup_size(const mfa_attention_kernel_t *kernel, uint32_t *out);
/** kernel.threadgroupMemoryAllocation  (:25, 272-363): dynamic shared memory bytes per CTA. */
MFA_API int mfa_attention_kernel_threadgroup_memory_allocation(const mfa_attention_kernel_t *kernel,
                                                               uint32_t *out);
/** Grid size the dispatch uses: ceil(parallelization dimension / blockDimensions.parallelization)
 *  (SquareAttentionTest.swift:328-339) times batch_count (dK/dV: times batch_count / kv_group, one CTA per K/V tile
 *  walks the query problems of its group). */
MFA_API int mfa_attention_kernel_grid_size(const mfa_attention_kernel_t *kernel,
                                           const mfa_function_constants_t *constants, uint32_t *out);
/** Name of the compiled kernel family ("attention_forward_tcgen05<128>" ...) -- stands in for
 *  kernel.createSource() (AttentionKernel+Source.swift:11-55), which has no analogue for
 *  ahead-of-time compiled CUDA.  Static storage owned by the kernel handle. */
MFA_API const char *mfa_attention_kernel_source_name(const mfa_attention_kernel_t *kernel);

/** What the reference leaves to its caller: makeLibrary + makeComputePipelineState + setBuffer x10
 *  + dispatchThreadgroups (SquareAttentionTest.swift:240-372).  `buffers[i]` is the DEVICE pointer
 *  bound at AttentionOperand.bufferBinding == i (Q0 K1 V2 O3 L4 D5 dO6 dV7 dK8 dQ9); slots the
 *  kernel type does not touch may be NULL.  Asynchronous on `cuda_stream` (a cudaStream_t, NULL =
 *  default stream).  Kernel order and dependencies are the reference's: forward writes O, L;
 *  backwardQuery reads O, L, dO and writes D, dQ; backwardKeyValue reads L, D and writes dK, dV
 *  (AttentionKernelType.swift:10-22).
 *  Some launches use a library-owned workspace per (device, stream): partial results of grids split across SMs, the
 *  zero-padded staging of head dimensions that are not multiples of 8, the FP16 copy of a BF16 dO.  It grows on demand
 *  with cudaMalloc, which is not possible while `cuda_stream` is being captured into a CUDA graph: encode the same
 *  problem size once outside the capture first (MFA_ERROR_CUDA with that message otherwise). */
MFA_API int mfa_attention_kernel_encode(const mfa_attention_kernel_t *kernel,
                                        const mfa_function_constants_t *constants,
                                        void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream);

/** Number of CUDA kernels one encode() launches.  Per slice of at most 16384 problems of the batch (a multiple of
 *  kv_group, so that a group never straddles two slices): 1; +1 when a small
 *  grid is split along the traversal axis and a merge kernel follows (split-KV combine for the forward, a plain sum of
 *  partial accumulators for dQ and dK/dV); +1 per operand staged row-major (head % 8 != 0 or stored transposed) and
 *  per output copied back from such a staging buffer; +1 when dK/dV converts a BF16 dO to FP16 in a pass of its own. */
MFA_API int mfa_attention_kernel_launch_count(const mfa_attention_kernel_t *kernel,
                                              const mfa_function_constants_t *constants, uint32_t *out);

/* ------------------------------------------------------------------------------------------ */
/* Variable-length (packed) sequences (library extension)                                      */
/* ------------------------------------------------------------------------------------------ */
/** One call over `count` sequences of different lengths: FlashAttention's cu_seqlens.  Sequence s owns query rows
 *  [row_offsets[s], row_offsets[s + 1]) and key rows [column_offsets[s], column_offsets[s + 1]) of every problem.  The
 *  buffers keep the layout of mfa_attention_kernel_encode, each problem contiguous: Q, O, dO, dQ are [batch_count][row]
 *  [D], L and D [batch_count][row], K, V, dK, dV [batch_count / kv_group][column][D], with row / column / batch_count /
 *  kv_group from the function constants (a packed [T, H, D] tensor is x.transpose(0, 1).contiguous(), row = T).
 *
 *  Within a sequence every output is exactly attention on that sequence: O, L, D, dQ of its Rs query rows over its Cs
 *  keys, and dK / dV summed over the query problems of each K/V group (deterministic, no atomics).  Causal is
 *  bottom-right aligned per sequence (delta = Cs - Rs).  A row that sees no key, including every row of a sequence
 *  with Cs = 0, gets O = 0, L = +inf, D = 0, dQ = 0; the keys of a sequence with Rs = 0 get dK = dV = 0.  Rows past
 *  row_offsets[count] / column_offsets[count] are never written, and the attention kernels do not read them (the
 *  staging copies of operands with head % 8 != 0 or a transposed layout, and the separate FP16 conversion of a BF16 dO,
 *  copy whole input buffers).  Packed calls never split a tile's traversal across CTAs.  MFA_BACKEND_SIMT_FP32 takes
 *  packed sequences with row-major operands only (MFA_ERROR_INVALID_ARGUMENT otherwise).
 *
 *  The offset tables are DEVICE memory, read by the kernels only (no host synchronisation; a packed encode can be
 *  captured into a CUDA graph and replayed with new table contents).  The host checks what it can see:
 *  MFA_ERROR_INVALID_ARGUMENT for a NULL table or offset pointer, count of 0 or above 65535 (the grid's z limit), and
 *  max_row / max_column of 0 or above row / column.  The kernels clamp every range into [0, row] / [0, column] (an end
 *  below its start counts as empty), so malformed contents never reach outside the caller's buffers; but a sequence
 *  longer than max_row / max_column breaks the contract: its rows past the maximum may be left unwritten. */
typedef struct mfa_sequence_table {
  uint32_t count;               /* S >= 1 */
  uint32_t max_row, max_column; /* host values >= every Rs / Cs: they size the grid */
  const int32_t *row_offsets;   /* device, S + 1 non-decreasing entries, last <= constants.row */
  const int32_t *column_offsets; /* device, S + 1 entries, last <= constants.column */
} mfa_sequence_table_t;
/** mfa_attention_kernel_encode over packed sequences. */
MFA_API int mfa_attention_kernel_encode_sequences(const mfa_attention_kernel_t *kernel,
                                                  const mfa_function_constants_t *constants,
                                                  const mfa_sequence_table_t *sequences,
                                                  void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream);
/** Grid size of a packed call: ceil(max_row (dK/dV: max_column) / parallelization) x problems x count. */
MFA_API int mfa_attention_kernel_grid_size_sequences(const mfa_attention_kernel_t *kernel,
                                                     const mfa_function_constants_t *constants,
                                                     const mfa_sequence_table_t *sequences, uint32_t *out);
/** Kernels one packed encode launches: as mfa_attention_kernel_launch_count, never with a split merge. */
MFA_API int mfa_attention_kernel_launch_count_sequences(const mfa_attention_kernel_t *kernel,
                                                        const mfa_function_constants_t *constants,
                                                        const mfa_sequence_table_t *sequences, uint32_t *out);

/* ------------------------------------------------------------------------------------------ */
/* Paged K/V cache (library extension; forward only)                                           */
/* ------------------------------------------------------------------------------------------ */
/** The forward over packed query sequences whose keys and values live in a paged cache, read in place: vLLM's block
 *  table, FlashAttention's flash_attn_with_kvcache(..., block_table=).  The pool is cut into pages of page_size = P
 *  key rows; sequence s owns the Cs keys whose pages page_table[s][0 .. ceil(Cs / P)) name, in order.
 *
 *  Layouts (function constants row, column, batch_count = H, kv_group = G):
 *    Q, O   [H][row][D] and L [H][row], as in a packed call: sequence s owns rows [row_offsets[s], row_offsets[s + 1]).
 *    K, V   page pools [num_pages][P][H / G][D] (the layout serving engines keep), column = num_pages * P pool rows.
 *           Key i of sequence s, K/V head kv, is pool row page_table[s][i / P] * P + i % P, head kv.
 *  Query head h reads K/V head h / G.  Within a sequence the output is attention of its Rs queries over its Cs keys;
 *  causal is bottom-right aligned per sequence (delta = Cs - Rs: the queries are the last Rs keys, which a decode or
 *  chunked-prefill step appends to the cache before the call).  A row that sees no key, including every row when
 *  Cs = 0, gets O = 0 and L = +inf.  Rows outside every sequence are never written.  Paged calls are never split.
 *
 *  The tables are DEVICE memory, read by the kernels only (a paged encode can be captured into a CUDA graph and
 *  replayed after column_lengths and page_table changed).  The host returns MFA_ERROR_INVALID_ARGUMENT, naming the
 *  field, for: a NULL table or device pointer; count of 0 or above 65535; max_row of 0 or above row; a page_size that
 *  is not a power of two, is below 16, or does not divide column; page_stride of 0; a backward kernel type; any
 *  transposed operand; on MFA_BACKEND_TCGEN05 a head dimension that is not a multiple of 8; batch_count above 16384
 *  (the pools interleave the heads of every token, so a batch is never sliced).  The kernels clamp what they read, so
 *  malformed contents never reach outside the caller's buffers: every query range as in mfa_sequence_table_t, every
 *  Cs into [0, page_stride * P] (no page-table row is read past its end), every page id into [0, num_pages).
 *  Page-table entries at or past ceil(Cs / P) are never read, and rows of a sequence's last page at or past Cs never
 *  reach its output (whatever they hold, NaN included).  As for packed calls, a sequence longer than max_row breaks
 *  the contract: its rows past the maximum may be left unwritten. */
typedef struct mfa_paged_kv {
  uint32_t count;                /* S >= 1 sequences */
  uint32_t max_row;              /* host value >= every Rs: sizes the grid */
  const int32_t *row_offsets;    /* device, S + 1 entries: the packed query rows, as mfa_sequence_table_t.row_offsets */
  const int32_t *column_lengths; /* device, S entries: Cs, the keys of sequence s (its cache length, new tokens included) */
  const int32_t *page_table;     /* device, [S][page_stride]: entry j holds the page of keys [j * P, (j + 1) * P) */
  uint32_t page_stride;          /* entries per page_table row */
  uint32_t page_size;            /* P: a power of two, >= 16, dividing column */
} mfa_paged_kv_t;
/** mfa_attention_kernel_encode of a forward kernel over a paged K/V cache. */
MFA_API int mfa_attention_kernel_encode_paged(const mfa_attention_kernel_t *kernel,
                                              const mfa_function_constants_t *constants, const mfa_paged_kv_t *paged,
                                              void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream);
/** Grid size of a paged call: ceil(max_row / parallelization) x batch_count x count. */
MFA_API int mfa_attention_kernel_grid_size_paged(const mfa_attention_kernel_t *kernel,
                                                 const mfa_function_constants_t *constants,
                                                 const mfa_paged_kv_t *paged, uint32_t *out);
/** Kernels one paged encode launches: 1. */
MFA_API int mfa_attention_kernel_launch_count_paged(const mfa_attention_kernel_t *kernel,
                                                    const mfa_function_constants_t *constants,
                                                    const mfa_paged_kv_t *paged, uint32_t *out);

/* ------------------------------------------------------------------------------------------ */
/* Sliding-window attention (library extension)                                                */
/* ------------------------------------------------------------------------------------------ */
/** A key band around the (bottom-right aligned) diagonal, FlashAttention's window_size: with delta = C - R, or Cs - Rs
 *  per sequence in packed and paged calls, query row i sees key j iff
 *      i + delta - left  <=  j  <=  i + delta + right,
 *  and a side of -1 has no bound.  A window of W keys ending at the diagonal is (W - 1, 0) on a causal kernel.  A row
 *  that sees no key gets O = 0, L = +inf, D = 0, dQ = 0, and a key that no row sees gets dK = dV = 0.  Every block
 *  and every page wholly outside the band is skipped: a paged forward never reads the page-table entries, nor loads the
 *  pages, whose keys lie outside the band of every query row of their sequence (for a causal (left, 0) window: the
 *  entries j with (j + 1) * P <= Cs - Rs - left), so a serving engine can recycle those pages. */
typedef struct mfa_attention_window {
  int32_t left, right; /* >= -1; a causal kernel takes right = 0 or -1 (both mean the diagonal) */
} mfa_attention_window_t;
/** mfa_attention_kernel_create of a kernel that applies `window`: every encode, grid-size and launch-count entry point
 *  (fixed, _sequences, _paged) honours it.  MFA_ERROR_INVALID_ARGUMENT, naming the field, for a NULL window, a value
 *  below -1, or right > 0 on a causal kernel.  The source name carries the window ("..._window<4095,0>"). */
MFA_API int mfa_attention_kernel_create_windowed(const mfa_attention_kernel_descriptor_t *kernel_descriptor,
                                                 const mfa_attention_window_t *window, mfa_attention_kernel_t **out);

/* ------------------------------------------------------------------------------------------ */
/* Split-KV decode (library extension; forward only)                                          */
/* ------------------------------------------------------------------------------------------ */
/** A forward over packed sequences or a paged cache whose key range may be split across CTAs, FlashAttention's
 *  flash_attn_with_kvcache(..., num_splits=).  A decode step has few query rows per sequence, so the unsplit grid of
 *  _sequences / _paged (one CTA per 128-row query tile, head and sequence) can leave most SMs idle while each CTA walks
 *  every key; the split grid gives each tile `splits` CTAs, each of which walks one key range and leaves a partial
 *  output that a second launch merges.
 *
 *  Buffer layouts, table contracts, window handling, empty rows (O = 0, L = +inf), rows outside every sequence (never
 *  written), the clamping of table contents and the isolation of NaN outside a sequence's keys are exactly those of
 *  mfa_attention_kernel_encode_sequences / _paged, and every check those calls make is made identically.  Beyond them,
 *  MFA_ERROR_INVALID_ARGUMENT, naming the field, for a NULL split, num_splits above 16, a backward kernel type
 *  ("only the forward"), and, in mfa_attention_kernel_split_plan, both or neither table.
 *
 *  The plan reads only host values: the kernel, the constants, the table's host fields and the hint.
 *    splits          num_splits when it is 1..16.  For 0: when the unsplit grid (tiles x batch_count x count) is at
 *                    most half the SMs, the most ranges up to SMs / grid and the parameter-table row's maximum (at most
 *                    16) whose ranges keep the row's minimum of key blocks (ceil(K / traversal block), K = the hint or
 *                    the table's bound, and for a windowed kernel at most the blocks the band of one tile meets); a
 *                    row whose minimum is 0 never splits.  On the device each tile's visible key blocks of its own
 *                    sequence are cut by ceiling into that many ranges; a range may be empty.
 *    heads_per_tile  kv_group when 2 <= kv_group <= 128 and max_row < 128 on the tensor cores (a tile then holds
 *                    floor(128 / kv_group) query rows of each query head of one K/V head, which reads each K/V block
 *                    once for the group instead of once per head), else 1.  The unsplit grid counts
 *                    ceil(max_row / rows per head) tiles x batch_count / heads_per_tile heads x count.
 *  A plan of one split and one head per tile launches the kernels of _sequences / _paged: the result, launches and
 *  grid are theirs, bit for bit.  One split with packed heads gives the same bits too (each row's arithmetic is that
 *  of the unpacked tile) in one launch.
 *  A split plan launches the split kernel and a merge (plus the operand staging of a packed call, as _sequences does).
 *  Split partials live in the per-(device, stream) workspace of the fixed-length split forward: encode a new size once
 *  outside a CUDA-graph capture first.  MFA_BACKEND_SIMT_FP32 accepts these calls and always plans one split, whatever
 *  num_splits says (its fixed-length calls do not split either). */
typedef struct mfa_split_kv {
  uint32_t num_splits; /* 0: the library's plan (above); 1..16: exactly this many key ranges per tile */
  uint32_t max_column; /* planning hint only: a bound on every Cs.  0 = the table's bound (max_column of a sequence
                          table; page_stride * P of a paged call).  Never a correctness contract: the key ranges are
                          cut on the device from each sequence's real Cs. */
} mfa_split_kv_t;

typedef struct mfa_split_plan {
  uint32_t splits;         /* key ranges per tile (1 = not split) */
  uint32_t heads_per_tile; /* 1, or kv_group when the query heads of one K/V head share a tile */
  uint32_t grid_size;      /* CTAs of the attention kernel */
  uint32_t launch_count;   /* kernels one encode launches */
} mfa_split_plan_t;

MFA_API int mfa_attention_kernel_encode_sequences_split(const mfa_attention_kernel_t *kernel,
                                                        const mfa_function_constants_t *constants,
                                                        const mfa_sequence_table_t *sequences,
                                                        const mfa_split_kv_t *split,
                                                        void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream);
MFA_API int mfa_attention_kernel_encode_paged_split(const mfa_attention_kernel_t *kernel,
                                                    const mfa_function_constants_t *constants,
                                                    const mfa_paged_kv_t *paged, const mfa_split_kv_t *split,
                                                    void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream);
/** The plan the two calls above follow; exactly one of sequences / paged non-NULL. */
MFA_API int mfa_attention_kernel_split_plan(const mfa_attention_kernel_t *kernel,
                                            const mfa_function_constants_t *constants,
                                            const mfa_sequence_table_t *sequences, const mfa_paged_kv_t *paged,
                                            const mfa_split_kv_t *split, mfa_split_plan_t *out);

/* ------------------------------------------------------------------------------------------ */
/* FP8 K/V cache (library extension; paged forward only)                                       */
/* ------------------------------------------------------------------------------------------ */
/** A paged forward (above) whose K and V pools hold one OCP FP8 E4M3 byte per element (torch.float8_e4m3fn: no
 *  infinities, NaN = 0x7F / 0xFF), [num_pages][P][H / G][D] bytes, the cache vLLM, SGLang, FlashInfer and
 *  TensorRT-LLM keep with kv_cache_dtype="fp8".  Key row i of K/V head kv stands for k_scale[kv] * e4m3(byte), and
 *  likewise for V with v_scale.  Q is FP16 or BF16 as the descriptor says; O is FP32 and L in the descriptor's precision.
 *
 *  The kernels dequantize on load: each FP8 value is converted exactly to Q's 16-bit type in shared memory, and the
 *  products, softmax and outputs are those of the 16-bit paged kernels.  k_scale[kv] multiplies the softmax scale and
 *  v_scale[kv] the output's normalisation, so with NULL scales, or scales that are powers of two, O and L equal bit for
 *  bit those of mfa_attention_kernel_encode_paged (split == NULL) or _paged_split (the same split) over the 16-bit pools
 *  holding the dequantized values.  Every guarantee of those calls holds unchanged: per-sequence causal alignment,
 *  grouped K/V, windows (pages outside the band are never read), split plans and packed query heads, empty rows
 *  (O = 0, L = +inf), the clamping of table contents, rows outside every sequence never written, pool contents past
 *  Cs never reaching an output (NaN bytes included), and graph replay as the cache grows.
 *
 *  The plan does not depend on the K/V element type: mfa_attention_kernel_grid_size_paged and _launch_count_paged
 *  describe an FP8 call with split == NULL, and mfa_attention_kernel_split_plan one with a split.
 *
 *  Every check of _paged (and, with a split, of _paged_split) is made identically.  Beyond them the host returns
 *  MFA_ERROR_INVALID_ARGUMENT, naming the field, before any device work for: a NULL fp8; a kernel on
 *  MFA_BACKEND_SIMT_FP32 ("FP8 K/V needs the tensor-core family"); a head dimension that is not a multiple of 16 (TMA
 *  reads 1-byte rows at 16-byte strides). */
typedef struct mfa_fp8_kv {
  const float *k_scale; /* device, batch_count / kv_group entries (one per K/V head), read at launch; NULL: every 1 */
  const float *v_scale; /* the same for V */
} mfa_fp8_kv_t;
/** split == NULL: as mfa_attention_kernel_encode_paged; else as mfa_attention_kernel_encode_paged_split. */
MFA_API int mfa_attention_kernel_encode_paged_fp8(const mfa_attention_kernel_t *kernel,
                                                  const mfa_function_constants_t *constants,
                                                  const mfa_paged_kv_t *paged, const mfa_split_kv_t *split,
                                                  const mfa_fp8_kv_t *fp8, void *const buffers[MFA_BUFFER_COUNT],
                                                  void *cuda_stream);

/* ------------------------------------------------------------------------------------------ */
/* Paged K/V append (library extension)                                                        */
/* ------------------------------------------------------------------------------------------ */
/** Writes a step's new keys and values into the page pools of a paged cache, through the table the paged forward reads
 *  (vLLM's reshape_and_cache).  With the mfa_paged_kv_t of the step:
 *    - sequence s owns new tokens [row_offsets[s], row_offsets[s + 1]) of k_new / v_new: Rs tokens;
 *    - column_lengths[s] is Cs, the sequence's length with the new tokens included, as the forward reads it;
 *    - new token i (0 <= i < Rs) becomes key p = Cs - Rs + i, pool row page_table[s][p / P] * P + p % P, every K/V head.
 *  This is the bottom-right alignment of the forward: an append followed by a paged encode on one stream attends over
 *  the cache with the step's tokens in it.
 *
 *  The kernel clamps as the forward does: row_offsets into [0, rows], Cs into [0, page_stride * P].  It never clamps a
 *  write: a position p < 0 (Rs > Cs) or a page id outside [0, pool_rows / P) is skipped.  So the append never writes
 *  outside k_pool / v_pool, nor a row the table does not name as one of the step's keys; tokens outside every sequence
 *  are never read.  As for the forward, a sequence longer than max_row breaks the contract: its tokens past max_row
 *  may be left unwritten.
 *
 *  fp8 == NULL: the pools hold `precision` elements ([num_pages][P][kv_heads][D]) and the append copies bit for bit.
 *  fp8 != NULL: the pools hold E4M3 bytes, as mfa_attention_kernel_encode_paged_fp8 reads them: element x of K/V head
 *  kv is stored as cvt.rn.satfinite.e4m3x2.f32(x / k_scale[kv]), x converted exactly to FP32 and / rounded to nearest
 *  (v_scale for V; a NULL scale is 1).  Finite values beyond +-448 and +-inf become +-448; NaN stays NaN.  That is
 *  torch's (x.float() / scale).clamp(-448, 448).to(torch.float8_e4m3fn), byte for byte.
 *
 *  One launch, no synchronisation, no allocation and no host read of device memory: the append can be captured into a
 *  CUDA graph with the forward and replayed after column_lengths / page_table changed in place.  The host returns
 *  MFA_ERROR_INVALID_ARGUMENT, naming the field, before any device work for: a NULL pointer (the table, its three
 *  device arrays, append, k_new, v_new, k_pool, v_pool); count of 0 or above 65535; max_row of 0 or above rows; a
 *  page_size that is not a power of two, is below 16, or does not divide pool_rows; page_stride of 0; kv_heads of 0;
 *  head_dimension of 0 or above 512; token_stride below kv_heads * head_dimension; an unknown precision.  Off sm_90 it
 *  returns MFA_ERROR_NO_DEVICE. */
typedef struct mfa_paged_kv_append {
  const void *k_new;       /* device: token t, K/V head kv, element d at element t * token_stride + kv * D + d */
  const void *v_new;       /* device: the same layout and stride */
  uint32_t rows;           /* T: tokens k_new / v_new hold (row_offsets are clamped into [0, T]) */
  uint32_t token_stride;   /* elements from one token to the next, >= kv_heads * D; 0 = kv_heads * D */
  uint32_t kv_heads;       /* Hkv >= 1 */
  uint32_t head_dimension; /* D, 1..512 */
  uint32_t pool_rows;      /* rows of each pool, num_pages * P: the forward's `column` */
  uint32_t precision;      /* mfa_precision_t of k_new / v_new: MFA_FP32, MFA_FP16 or MFA_BF16 */
} mfa_paged_kv_append_t;   /* 40 bytes */

MFA_API int mfa_paged_kv_append(const mfa_paged_kv_t *paged, const mfa_paged_kv_append_t *append, void *k_pool,
                                void *v_pool, const mfa_fp8_kv_t *fp8, void *cuda_stream);

/* ------------------------------------------------------------------------------------------ */
/* Rotary append (library extension)                                                           */
/* ------------------------------------------------------------------------------------------ */
/** mfa_paged_kv_append with rotary position embedding (RoPE), FlashAttention's rotary_cos / rotary_sin of
 *  flash_attn_with_kvcache: the step's queries and new keys are rotated at their cache positions, and the queries are
 *  written in the paged forward's Q layout, in one launch.
 *
 *  New token i of sequence s sits at position p = Cs - Rs + i: the key mfa_paged_kv_append writes, with the same
 *  clamping of query ranges and Cs.  With c = cos[p][j] and s = sin[p][j], each pair (x, y) of q (every query head) and
 *  of k (every K/V head) becomes x' = x c - y s, y' = y c + x s: x, y converted exactly to FP32, each product and the
 *  sum or difference rounded separately (no FMA), the result rounded to nearest-even to append->precision (FP32 stays
 *  FP32).  Pairs are (j, j + r/2) (GPT-NeoX / Llama rotate_half) or, interleaved, (2j, 2j + 1) (GPT-J), for
 *  0 <= j < r/2.  Elements d >= r and V pass through unchanged.  FP8 pools receive the rounded rotated k quantized
 *  exactly as mfa_paged_kv_append quantizes a source value.  So k_pool / v_pool hold the bytes mfa_paged_kv_append
 *  writes for rope(k_new) and v_new, and q_out holds rope(q_new) transposed to [query_heads][rows][D], with rope
 *  torch's (x.float() * c - y.float() * s).to(dtype), op by op.
 *
 *  Row (h, q0 + i) of q_out is written iff p >= 0: rows of tokens with p < 0 (Rs > Cs) and rows outside every sequence
 *  are never written.  A K/V row is written under mfa_paged_kv_append's rule.  Scaled RoPE variants (linear, NTK,
 *  YaRN, Llama-3) live in the tables.  vLLM's cos_sin_cache [max_pos][r] (cos half, then sin half) is passed as
 *  cos = base, sin = base + r/2, table_stride = r; FlashAttention's [seqlen][r/2] tables use table_stride 0.
 *
 *  No synchronisation, allocation or host read of device memory: the call captures into a CUDA graph with the split
 *  forward and replays as column_lengths / page_table change in place.  q_new and q_out must not overlap.
 *
 *  Every check of mfa_paged_kv_append is made first, identically.  Beyond them the host returns
 *  MFA_ERROR_INVALID_ARGUMENT, naming the field, before any device work for: a NULL rotary, q_new, q_out, cos or sin;
 *  query_heads of 0 or not a multiple of kv_heads; query_heads * D above 2^32 - 1; a nonzero q_token_stride below
 *  query_heads * D; rotary_dim of 0, odd or above D; a nonzero table_stride below r / 2; positions below
 *  page_stride * page_size (so the kernel never reads past the tables); interleaved other than 0 or 1.  Off sm_90 it
 *  returns MFA_ERROR_NO_DEVICE. */
typedef struct mfa_rotary {
  const void *q_new;       /* device: token t, query head h, element d at t * q_token_stride + h * D + d; append->precision */
  void *q_out;             /* device: the paged forward's Q buffer, [query_heads][append->rows][D]; append->precision */
  const float *cos;        /* device FP32: position p, frequency j (0 <= j < rotary_dim / 2) at p * table_stride + j */
  const float *sin;        /* the same layout */
  uint32_t query_heads;    /* H: a multiple of append->kv_heads (the forward's batch_count) */
  uint32_t q_token_stride; /* elements from one token to the next, >= query_heads * D; 0 = query_heads * D */
  uint32_t rotary_dim;     /* r: even, 2..D; elements d >= r pass through unchanged (partial rotary) */
  uint32_t table_stride;   /* floats per table row, >= r / 2; 0 = r / 2 */
  uint32_t positions;      /* rows of cos / sin: at least page_stride * page_size */
  uint32_t interleaved;    /* 0: pairs (j, j + r/2) (GPT-NeoX / Llama rotate_half); 1: pairs (2j, 2j + 1) (GPT-J) */
} mfa_rotary_t;            /* 56 bytes */

MFA_API int mfa_paged_kv_append_rotary(const mfa_paged_kv_t *paged, const mfa_paged_kv_append_t *append,
                                       const mfa_rotary_t *rotary, void *k_pool, void *v_pool,
                                       const mfa_fp8_kv_t *fp8, void *cuda_stream);

/* ------------------------------------------------------------------------------------------ */
/* Kernel cache keyed by descriptor                                                            */
/* ------------------------------------------------------------------------------------------ */
/** The analogue of the reference's pipeline cache (GEMMKernel.register(descriptor:) / pipelineCache[descriptor],
 *  R/GEMM/GEMMDescriptor/GEMMDescriptor+PipelineCache.swift:16-36): descriptor.kernelDescriptor(type:) +
 *  AttentionKernel(descriptor:) run once per distinct (descriptor, type) and the validated kernel object is kept.
 *  R, C and batch_count are launch-time constants and not part of the key.  The returned handle is owned by the
 *  library (do NOT destroy it), is immutable, and stays valid until the process exits.  Thread-safe. */
MFA_API int mfa_attention_kernel_cache_fetch(const mfa_attention_descriptor_t *descriptor, mfa_kernel_type_t type,
                                             const mfa_attention_kernel_t **out);
/** mfa_attention_kernel_cache_fetch of a windowed kernel (mfa_attention_kernel_create_windowed), keyed by
 *  (descriptor, type, window): the same window returns the same handle. */
MFA_API int mfa_attention_kernel_cache_fetch_windowed(const mfa_attention_descriptor_t *descriptor,
                                                      mfa_kernel_type_t type, const mfa_attention_window_t *window,
                                                      const mfa_attention_kernel_t **out);
/** Number of kernel objects the cache currently holds. */
MFA_API int mfa_attention_kernel_cache_size(void);

/* ------------------------------------------------------------------------------------------ */
/* Host-buffer convenience (the e2e path): H2D -> selected kernels -> D2H, synchronous.        */
/* ------------------------------------------------------------------------------------------ */
#define MFA_RUN_FORWARD (1u << MFA_FORWARD)
#define MFA_RUN_BACKWARD_QUERY (1u << MFA_BACKWARD_QUERY)
#define MFA_RUN_BACKWARD_KEY_VALUE (1u << MFA_BACKWARD_KEY_VALUE)

/** `host_buffers[i]` are HOST pointers laid out exactly like the device buffers (element type =
 *  memoryPrecisions[operand]).  Inputs (Q,K,V, and dO for backward) are copied to the device,
 *  the kernels in `run_mask` are encoded in the reference's order fwd -> dQ -> dK/dV, and every
 *  output they produce whose host pointer is non-NULL is copied back.  Device scratch is owned
 *  by the library (grown on demand, one set per calling thread and device).  `device` = CUDA device
 *  ordinal; the caller's current device is restored before the call returns.
 *  With batch_count > 1 the independent problems are processed in chunks that rotate over three
 *  streams, so uploads, kernels and downloads of neighbouring chunks overlap (pass page-locked host
 *  memory to get the overlap; pageable memory still works, serialised by the driver).
 *  Every problem has its own K and V here (kv_group = 1): grouped K/V goes through mfa_attention_kernel_encode.
 *  There is no window here either: a sliding window goes through mfa_attention_kernel_create_windowed /
 *  mfa_attention_kernel_cache_fetch_windowed and mfa_attention_kernel_encode. */
MFA_API int mfa_attention_run_host(const mfa_attention_descriptor_t *descriptor, uint32_t run_mask,
                                   void *const host_buffers[MFA_BUFFER_COUNT], int device);

/* Host-memory placement for the host-buffer path (library extension; the reference's buffers are Metal shared-storage
 * buffers, MTLContext+Buffers.swift:5-45, with no placement to speak of on a unified-memory SoC). */
/** Page-locked host buffer for mfa_attention_run_host, allocated (first-touched) on the NUMA node `device` hangs
 *  off and portable across CUDA contexts.  The calling thread's CPU affinity is unchanged on return. */
MFA_API int mfa_host_alloc(size_t bytes, int device, void **out);
/** The same for buffers the host only WRITES and the GPU reads (Q, K, V, dO of mfa_attention_run_host): the pages are also
 *  write-combined, so the upload's PCIe reads are not snooped through the CPU caches and the buffers do not evict the
 *  host's working set.  Reading such a buffer with the CPU is very slow: do not use it for outputs. */
MFA_API int mfa_host_alloc_upload(size_t bytes, int device, void **out);
MFA_API int mfa_host_free(void *ptr);
/** Restricts the calling thread to the CPUs of `device`'s NUMA node (within the affinity it already has), so that
 *  memory it allocates afterwards and the copies it issues stay on the GPU's socket.  `*numa_node` (optional) receives
 *  the node, or -1 when the platform reports none (then nothing is changed). */
MFA_API int mfa_host_bind_thread_to_device(int device, int *numa_node);

/** Frees what the library holds on `device`: the calling thread's run_host scratch (operand buffers, streams, events)
 *  and every split-grid workspace of the device.  Synchronises the device first.  Optional -- everything is reused
 *  across calls and reclaimed at process exit; long-lived hosts that are done with a device call this. */
MFA_API int mfa_release_device_resources(int device);

/** Element count of operand's buffer for one problem (R*D, C*D, R ...) times batch_count. */
MFA_API int mfa_attention_descriptor_operand_elements(const mfa_attention_descriptor_t *descriptor,
                                                      mfa_operand_t operand, size_t *out);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* MFA_B200_H */
