// AttentionDescriptor side of the C ABI: precision policy, H100 parameter tables, and the
// descriptor -> kernel-descriptor heuristic.  Mirrors (does not copy) the reference's
//   Sources/FlashAttention/Attention/AttentionDescriptor/AttentionDescriptor.swift
//   .../AttentionDescriptor+Precisions.swift, +Parameters.swift, AttentionParameterRow.swift
// The tables hold H100 tile shapes and on-chip residency instead of Apple register-cache choices.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "internal.h"

namespace mfa {
constexpr int kTableSlots = 6;  // parameter tables of the tensor-core family (see table_slot)

thread_local std::string g_last_error;

int fail(int status, const std::string &message) {
  g_last_error = message;
  return status;
}

static const char *kOperandNames[MFA_OPERAND_COUNT] = {"Q",  "K",  "V",  "O",  "L", "D",  "dO",
                                                       "dV", "dK", "dQ", "S",  "P", "dP", "dS"};

// ------------------------------------------------------------------------------------------------
// Precision policy
// ------------------------------------------------------------------------------------------------

// memoryPrecisions (AttentionDescriptor+Precisions.swift:10-146)
int memory_precision(const mfa_attention_descriptor_t &d, int operand) {
  const bool bf16Inputs = d.input_precision_override == MFA_BF16;
  switch (operand) {
    case MFA_Q: case MFA_K: case MFA_V:
      // :13-23  FP16 when lowPrecisionInputs (extension: BF16 when overridden)
      return d.low_precision_inputs ? (bf16Inputs ? MFA_BF16 : MFA_FP16) : MFA_FP32;
    case MFA_dO:
      // :17,22  BF16 when lowPrecisionInputs (extension: FP16 when the override asks for an all-FP16 operand set)
      return d.low_precision_inputs ? (d.input_precision_override == MFA_FP16 ? MFA_FP16 : MFA_BF16) : MFA_FP32;
    case MFA_L:
      return d.low_precision_intermediates ? MFA_FP16 : MFA_FP32;  // :81-87
    case MFA_D:
      return d.low_precision_intermediates ? MFA_BF16 : MFA_FP32;
    case MFA_O: case MFA_dV: case MFA_dK: case MFA_dQ:
      return MFA_FP32;  // :140-143  always FP32 in memory
    default:
      return -1;  // S, P, dP, dS are never materialised
  }
}

// registerPrecisions (AttentionDescriptor+Precisions.swift:149-215).  H100 has native BF16
// conversion, so the `hasNativeBF16Casting` (Apple9) branch applies.  `type` selects the kernel whose registers are
// described: the precision of P and dS depends on the kernel family that serves (descriptor, type) -- on the tensor-core
// family they are operands of a tensor-core MMA and therefore ALWAYS carried in the 16-bit input element type, whatever
// lowPrecisionIntermediates says (the reference keeps them in FP32 registers when that flag is off, :203-205; this is a
// documented deviation, DESIGN.md section 3, and the descriptor reports what the kernel really does).
int register_precision_for(const mfa_attention_descriptor_t &d, int operand, int type) {
  const bool bf16Inputs = d.input_precision_override == MFA_BF16;
  const bool tensorCore = select_backend(d, type) == MFA_BACKEND_TCGEN05;
  switch (operand) {
    case MFA_Q: case MFA_K: case MFA_V:
      return d.low_precision_inputs ? (bf16Inputs ? MFA_BF16 : MFA_FP16) : MFA_FP32;  // :158-168
    case MFA_dO:
      return d.low_precision_inputs ? (d.input_precision_override == MFA_FP16 ? MFA_FP16 : MFA_BF16) : MFA_FP32;
    case MFA_L:
      return d.low_precision_intermediates ? MFA_FP16 : MFA_FP32;  // :171-177
    case MFA_D:
      return d.low_precision_intermediates ? MFA_BF16 : MFA_FP32;
    case MFA_S:
      // :197  S accumulates in FP16 only when both flags are set.  H100 tensor cores always
      // accumulate S in FP32 (wgmma accumulators), which is the more accurate of the two; report FP32.
      return MFA_FP32;
    case MFA_P:
      // :198  P is a 16-bit value under lowPrecisionIntermediates; on the tensor-core family it is always rounded to the
      // input element type (it is the A operand of O += P V, dV += P^T dO)
      if (tensorCore || d.low_precision_intermediates) return bf16Inputs ? MFA_BF16 : MFA_FP16;
      return MFA_FP32;
    case MFA_dP:
      return MFA_FP32;  // :199
    case MFA_dS:
      // :200  BF16 under lowPrecisionIntermediates (Apple9); on the tensor-core family the A operand of dQ += dS K,
      // dK += dS^T Q, in the input element type
      if (tensorCore) return bf16Inputs ? MFA_BF16 : MFA_FP16;
      return d.low_precision_intermediates ? MFA_BF16 : MFA_FP32;
    case MFA_O: case MFA_dV: case MFA_dK: case MFA_dQ:
      return MFA_FP32;  // :209-212  all outputs accumulate in FP32
    default:
      return -1;
  }
}

// descriptor-level view (no kernel type in the reference's API): P as the forward kernel holds it, dS as backwardQuery
int register_precision(const mfa_attention_descriptor_t &d, int operand) {
  return register_precision_for(d, operand, operand == MFA_dS ? MFA_BACKWARD_QUERY : MFA_FORWARD);
}

// ------------------------------------------------------------------------------------------------
// H100 parameter tables.  Same text format as the reference's "parameter file"
// (AttentionDescriptor+Parameters.swift:106-285):
//     | max head dimension | parallelization | traversal | head block | resident operands |
// First row with D <= max wins (:41-66); past the end, the last row applies.
//   * tensor-core family: parallelization = Q (or K/V) rows per CTA, traversal = keys (queries) per pipeline
//     stage, head block = the padded head dimension (accumulators in registers up to 256), resident = operands
//     that stay in shared memory / registers for the entire traversal.
//   * SIMT family: 64 x 64 blocks, 32-wide head chunks, accumulators resident in registers.
// ------------------------------------------------------------------------------------------------
// Tensor-core rows carry two tuning columns after the reference's five:
//     | min blocks per split | max splits |
// They govern small grids: the forward cuts every query tile's key axis into equal ranges of at least `min blocks`
// key blocks and merges the partials (split-KV); the backward kernels cut their traversal axis likewise and sum the
// partial gradients.  0 min blocks turns splitting off.
//   forward: 128 query rows per CTA (two warpgroups); 128-key blocks up to D = 128, 64-key blocks beyond
//   backwardQuery: 128 query rows per CTA up to D = 128, 64 beyond (one warpgroup); 64-key blocks
//   backwardKeyValue: 128 key rows per CTA up to D = 128, 64 beyond (dK / dV columns split over two warpgroups);
//   64-query blocks
// Transposed operands are staged row-major first and run the same kernels.
static const char *kForwardWgmma =
    "| 64  | 128 | 128 | 64  | Q, O | 2 | 8 |\n"
    "| 128 | 128 | 128 | 128 | Q, O | 4 | 8 |\n"
    "| 256 | 128 | 64  | 256 | Q, O | 0 | 1 |\n"
    "\n";
static const char *kForwardWgmmaTransposed =
    "| 64  | 128 | 128 | 64  | Q, O | 0 | 1 |\n"
    "| 128 | 128 | 128 | 128 | Q, O | 0 | 1 |\n"
    "| 256 | 128 | 64  | 256 | Q, O | 0 | 1 |\n"
    "\n";
static const char *kBackwardQueryWgmma =
    "| 64  | 128 | 64  | 64  | Q, dO, dQ | 2 | 8 |\n"
    "| 128 | 128 | 64  | 128 | Q, dO, dQ | 2 | 8 |\n"
    "| 256 | 64  | 64  | 256 | Q, dO, dQ | 2 | 8 |\n"
    "\n";
static const char *kBackwardKeyValueWgmma =
    "| 64  | 128 | 64  | 64  | K, V, dV, dK | 2 | 8 |\n"
    "| 128 | 128 | 64  | 128 | K, V, dV, dK | 2 | 8 |\n"
    "| 256 | 64  | 64  | 256 | K, V, dV, dK | 2 | 8 |\n"
    "\n";
static const char *kBackwardQueryWgmmaTransposed = kBackwardQueryWgmma;
static const char *kBackwardKeyValueWgmmaTransposed = kBackwardKeyValueWgmma;
static const char *kForwardSimt =
    "| 512 | 64 | 64 | 32 | O |\n"
    "\n";
static const char *kBackwardQuerySimt =
    "| 512 | 64 | 64 | 32 | dQ |\n"
    "\n";
static const char *kBackwardKeyValueSimt =
    "| 256 | 64 | 64 | 32 | dV, dK |\n"
    "| 512 | 64 | 64 | 32 |        |\n"
    "\n";

// Which kernel family can serve this descriptor.  The tensor-core family needs 16-bit operands; its kernels read
// row-major operands with D % 8 == 0 (TMA global-stride rule), anything else is staged into that form first.
static bool any_transpose(const mfa_attention_descriptor_t &d) {
  return d.transpose_Q || d.transpose_K || d.transpose_V || d.transpose_O;
}

// Transposed operands are staged row-major where the transposed view has a 16-byte row pitch (sequence length % 8 ==
// 0): Q^T and (backward only) dO^T, which follows O, are addressed through R, K^T and V^T through C.
static bool transposes_ok(const mfa_attention_descriptor_t &d, int type) {
  return (!d.transpose_Q || d.row % 8 == 0) && (!d.transpose_K || d.column % 8 == 0) &&
         (!d.transpose_V || d.column % 8 == 0) && (type == MFA_FORWARD || !d.transpose_O || d.row % 8 == 0);
}

int select_backend(const mfa_attention_descriptor_t &d, int type) {
  if (!d.low_precision_inputs || d.head == 0) return MFA_BACKEND_SIMT_FP32;
  const uint32_t padded = (static_cast<uint32_t>(d.head) + 7) / 8 * 8;
  if (any_transpose(d)) {
    if (!transposes_ok(d, type)) return MFA_BACKEND_SIMT_FP32;
    if (d.head % 8 != 0) return MFA_BACKEND_SIMT_FP32;  // (head-dimension padding is implemented for row-major operands)
  }
  // D % 8 != 0 (row-major): the operands are staged with pad8(D) columns (kernels/pad_head.cu) and the tensor-core kernels
  // run at the padded head dimension -- the reference's zero-padded async copies (+OuterProduct.swift:237-254)
  if (padded > kWgmmaMaxHead) return MFA_BACKEND_SIMT_FP32;
  // (the reference's own policy, FP16 Q/K/V + BF16 dO, is served too: wgmma cannot mix element types
  // inside one MMA, so the backward kernels rewrite the staged dO tile as FP16 in shared memory)
  return MFA_BACKEND_TCGEN05;
}

// The tensor-core tables are data: mfa_set_parameter_table() / MFA_B200_PARAMETER_FILE replace them at run time.
// slot 0 forward, 2 backwardQuery, 4 backwardKeyValue; +1: the table used with transposed operands; empty = built-in
static std::string g_table_override[kTableSlots];
static bool g_table_overridden[kTableSlots] = {false, false, false, false, false, false};
static unsigned g_table_generation = 0;
unsigned parameter_table_generation() { return g_table_generation; }

static const char *builtin_table(int slot) {
  switch (slot) {
    case 0: return kForwardWgmma;
    case 1: return kForwardWgmmaTransposed;
    case 2: return kBackwardQueryWgmma;
    case 3: return kBackwardQueryWgmmaTransposed;
    case 4: return kBackwardKeyValueWgmma;
    default: return kBackwardKeyValueWgmmaTransposed;
  }
}
static int table_slot(int type, bool transposed) {
  return (type == MFA_FORWARD ? 0 : (type == MFA_BACKWARD_QUERY ? 2 : 4)) + (transposed ? 1 : 0);
}

const char *parameter_file(const mfa_attention_descriptor_t &d, int type) {
  const bool tc = select_backend(d, type) == MFA_BACKEND_TCGEN05;
  if (tc) {
    const int slot = table_slot(type, any_transpose(d));
    return g_table_overridden[slot] ? g_table_override[slot].c_str() : builtin_table(slot);
  }
  switch (type) {
    case MFA_FORWARD: return kForwardSimt;
    case MFA_BACKWARD_QUERY: return kBackwardQuerySimt;
    default: return kBackwardKeyValueSimt;
  }
}

// AttentionParameterRow (AttentionParameterRow.swift:8-19)
struct ParameterRow {
  unsigned maximumHeadDimension = 0;
  std::string parallelization, traversal, head, cachedOperands;
  // tuning columns (present in the tensor-core tables; empty = defaults)
  std::string splitMinBlocks, splitMax;
};

static std::string strip_spaces(const std::string &s) {
  std::string out;
  for (char c : s)
    if (c != ' ') out.push_back(c);  // AttentionParameterRow.swift:39-41 removes 0x20 only
  return out;
}

// parseTable (AttentionParameterRow.swift:22-74)
static int parse_table(const char *file, std::vector<ParameterRow> &rows) {
  std::string text(file);
  size_t pos = 0;
  while (pos < text.size()) {
    size_t eol = text.find('\n', pos);
    if (eol == std::string::npos) eol = text.size();
    std::string line = text.substr(pos, eol - pos);
    pos = eol + 1;
    if (line.empty()) continue;  // Swift's split(separator:) omits empty subsequences
    std::vector<std::string> segments;
    size_t p = 0;
    while (p <= line.size()) {
      size_t bar = line.find('|', p);
      if (bar == std::string::npos) bar = line.size();
      std::string seg = line.substr(p, bar - p);
      if (!seg.empty()) segments.push_back(strip_spaces(seg));
      p = bar + 1;
    }
    if (segments.size() != 5 && segments.size() != 7)  // the reference's five columns, or five + two tuning columns
      return fail(MFA_ERROR_INVALID_ARGUMENT, "Number of segments was invalid: " + std::to_string(segments.size()));
    ParameterRow row;
    char *end = nullptr;
    unsigned long maxHead = strtoul(segments[0].c_str(), &end, 10);
    if (segments[0].empty() || *end != '\0' || maxHead > 65535)
      return fail(MFA_ERROR_INVALID_ARGUMENT, "Could not extract maximum head dimension.");
    row.maximumHeadDimension = static_cast<unsigned>(maxHead);
    row.parallelization = segments[1];
    row.traversal = segments[2];
    row.head = segments[3];
    row.cachedOperands = segments[4];
    if (segments.size() == 7) {
      row.splitMinBlocks = segments[5];
      row.splitMax = segments[6];
    }
    rows.push_back(row);
  }
  return MFA_SUCCESS;
}

// parseOperands (AttentionParameterRow.swift:76-106)
static int parse_operands(const std::string &text, std::vector<int> &operands) {
  static const int accepted[] = {MFA_Q, MFA_K, MFA_V, MFA_O, MFA_dO, MFA_dV, MFA_dK, MFA_dQ};
  size_t p = 0;
  while (p <= text.size()) {
    size_t comma = text.find(',', p);
    if (comma == std::string::npos) comma = text.size();
    std::string name = text.substr(p, comma - p);
    p = comma + 1;
    if (name.empty()) continue;
    int matched = -1;
    for (int op : accepted)
      if (name == kOperandNames[op]) matched = op;
    if (matched < 0) return fail(MFA_ERROR_INVALID_ARGUMENT, "Could not find match for " + name + ".");
    operands.push_back(matched);
  }
  return MFA_SUCCESS;
}

static bool parse_u16(const std::string &s, uint16_t &out) {
  if (s.empty()) return false;
  char *end = nullptr;
  unsigned long v = strtoul(s.c_str(), &end, 10);
  if (*end != '\0' || v > 65535) return false;
  out = static_cast<uint16_t>(v);
  return true;
}

// kernelDescriptor(type:)  (AttentionDescriptor.swift:33-130)
int kernel_descriptor(const mfa_attention_descriptor_t &d, int type, mfa_attention_kernel_descriptor_t &out) {
  if (type < MFA_FORWARD || type > MFA_BACKWARD_KEY_VALUE)
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Unrecognized kernel type.");
  // createHeadDimension / createTransposeState guard clauses (:88-111)
  if (!d.has_matrix_dimensions || !d.has_transpose_state)
    return fail(MFA_ERROR_INCOMPLETE_DESCRIPTOR, "Descriptor was incomplete.");
  if (d.causal > 1) return fail(MFA_ERROR_INVALID_ARGUMENT, "Unrecognized causal mask mode.");

  // Fetch the kernel-specific parameters (:36-39).
  std::vector<ParameterRow> table;
  int status = parse_table(parameter_file(d, type), table);
  if (status != MFA_SUCCESS) return status;
  // row(table:)  (AttentionDescriptor+Parameters.swift:41-66): first row with D <= max, else the last.
  const ParameterRow *row = &table.back();
  for (const ParameterRow &candidate : table) {
    if (d.head <= candidate.maximumHeadDimension) {
      row = &candidate;
      break;
    }
  }

  mfa_attention_kernel_descriptor_init(&out);

  // createBlockDimensions (:41-54): head block <= pad8(D)
  uint16_t parallelization, traversal, originalHead;
  if (!parse_u16(row->parallelization, parallelization) || !parse_u16(row->traversal, traversal) ||
      !parse_u16(row->head, originalHead))
    return fail(MFA_ERROR_INVALID_ARGUMENT, "Could not decode block dimensions.");
  const uint16_t paddedHeadDimension = static_cast<uint16_t>((d.head + 7) / 8 * 8);
  out.has_block_dimensions = 1;
  out.block_parallelization = parallelization;
  out.block_traversal = traversal;
  out.block_head = originalHead < paddedHeadDimension ? originalHead : paddedHeadDimension;

  // createCacheState (:56-86)
  uint16_t expected = 0;
  switch (type) {
    case MFA_FORWARD: expected = (1u << MFA_Q) | (1u << MFA_O); break;
    case MFA_BACKWARD_QUERY: expected = (1u << MFA_Q) | (1u << MFA_dO) | (1u << MFA_dQ); break;
    default: expected = (1u << MFA_K) | (1u << MFA_V) | (1u << MFA_dV) | (1u << MFA_dK); break;
  }
  std::vector<int> cached;
  status = parse_operands(row->cachedOperands, cached);
  if (status != MFA_SUCCESS) return status;
  uint16_t cachedMask = 0;
  for (int operand : cached) {
    if (!(expected & (1u << operand)))
      return fail(MFA_ERROR_UNEXPECTED_OPERAND, std::string("Unexpected operand: ") + kOperandNames[operand]);
    cachedMask |= (1u << operand);
  }
  out.cache_state_valid_mask = expected;
  out.cache_state_mask = cachedMask;

  out.has_head_dimension = 1;
  out.head_dimension = d.head;

  for (int operand = 0; operand < MFA_OPERAND_COUNT; ++operand) {
    int mem = memory_precision(d, operand);
    int reg = register_precision_for(d, operand, type);
    out.memory_precisions[operand] = mem < 0 ? 0xFF : static_cast<uint8_t>(mem);
    out.register_precisions[operand] = reg < 0 ? 0xFF : static_cast<uint8_t>(reg);
  }

  out.backend = static_cast<uint8_t>(select_backend(d, type));
  // tuning columns (tensor-core tables); rows without them (the FP32 family) leave the default: no splits
  out.split_min_blocks = 0;
  out.split_max = 1;
  if (!row->splitMinBlocks.empty()) {
    uint16_t minBlocks = 0, maxSplits = 0;
    if (!parse_u16(row->splitMinBlocks, minBlocks) || !parse_u16(row->splitMax, maxSplits) || minBlocks > 255 ||
        maxSplits > 255)
      return fail(MFA_ERROR_INVALID_ARGUMENT, "Could not decode tuning columns.");
    out.split_min_blocks = static_cast<uint8_t>(minBlocks);
    out.split_max = static_cast<uint8_t>(maxSplits < 1 ? 1 : maxSplits);
  }
  // preferAsyncCache / preferAsyncLoad (:118-124): "async" == TMA bulk-tensor copies on H100.
  out.prefer_async_cache = out.backend == MFA_BACKEND_TCGEN05 ? 1 : 0;
  out.prefer_async_load = out.backend == MFA_BACKEND_TCGEN05 ? 1 : 0;

  // createTransposeState (:96-111): derivatives follow their forward operand.
  uint16_t t = 0;
  if (d.transpose_Q) t |= (1u << MFA_Q) | (1u << MFA_dQ);
  if (d.transpose_K) t |= (1u << MFA_K) | (1u << MFA_dK);
  if (d.transpose_V) t |= (1u << MFA_V) | (1u << MFA_dV);
  if (d.transpose_O) t |= (1u << MFA_O) | (1u << MFA_dO);
  out.transpose_state_valid_mask = (1u << MFA_Q) | (1u << MFA_K) | (1u << MFA_V) | (1u << MFA_O) | (1u << MFA_dO) |
                                   (1u << MFA_dV) | (1u << MFA_dK) | (1u << MFA_dQ);
  out.transpose_state_mask = t;
  out.type = static_cast<uint8_t>(type);
  out.causal = d.causal;
  return MFA_SUCCESS;
}

}  // namespace mfa

// MFA_B200_PARAMETER_FILE: tables from a file, installed when the library is loaded.  Sections "[forward]",
// "[forward.transposed]", "[backwardQuery]", "[backwardKeyValue]"; lines starting with '#' are comments.  A malformed
// section is reported on stderr and skipped (the built-in table stays).
namespace {
struct ParameterFileLoader {
  ParameterFileLoader() {
    const char *path = getenv("MFA_B200_PARAMETER_FILE");
    if (!path || !*path) return;
    FILE *f = fopen(path, "r");
    if (!f) {
      fprintf(stderr, "mfa_b200: cannot open MFA_B200_PARAMETER_FILE=%s\n", path);
      return;
    }
    static const char *names[mfa::kTableSlots] = {"[forward]", "[forward.transposed]", "[backwardQuery]",
                                             "[backwardQuery.transposed]", "[backwardKeyValue]", "[backwardKeyValue.transposed]"};
    static const int types[mfa::kTableSlots] = {MFA_FORWARD, MFA_FORWARD, MFA_BACKWARD_QUERY, MFA_BACKWARD_QUERY,
                                           MFA_BACKWARD_KEY_VALUE, MFA_BACKWARD_KEY_VALUE};
    std::string text[mfa::kTableSlots];
    int current = -1;
    char line[1024];
    while (fgets(line, sizeof(line), f)) {
      std::string l(line);
      while (!l.empty() && (l.back() == '\n' || l.back() == '\r' || l.back() == ' ')) l.pop_back();
      if (l.empty() || l[0] == '#') continue;
      if (l[0] == '[') {
        current = -1;
        for (int i = 0; i < mfa::kTableSlots; ++i)
          if (l == names[i]) current = i;
        continue;
      }
      if (current >= 0) text[current] += l + "\n";
    }
    fclose(f);
    for (int i = 0; i < mfa::kTableSlots; ++i)
      if (!text[i].empty() &&
          mfa_set_parameter_table(static_cast<mfa_kernel_type_t>(types[i]), i & 1, text[i].c_str()) != MFA_SUCCESS)
        fprintf(stderr, "mfa_b200: section %s of %s rejected: %s\n", names[i], path, mfa_last_error());
  }
} g_parameter_file_loader;
}  // namespace

// ------------------------------------------------------------------------------------------------
// extern "C" surface
// ------------------------------------------------------------------------------------------------
using namespace mfa;

extern "C" {

const char *mfa_last_error(void) { return g_last_error.c_str(); }
const char *mfa_version(void) { return "mfa_b200 0.5 (sm_90a; wgmma+TMA forward / dQ / dK-dV, SIMT FP32 family, grouped K/V, packed sequences, paged K/V, sliding window, split-KV decode, FP8 K/V, paged K/V append, rotary append)"; }

int mfa_precision_size(mfa_precision_t precision) { return precision == MFA_FP32 ? 4 : 2; }
const char *mfa_precision_name(mfa_precision_t precision) {
  switch (precision) {
    case MFA_FP32: return "float";
    case MFA_FP16: return "half";
    case MFA_BF16: return "bfloat";
  }
  return "";
}

const char *mfa_operand_name(mfa_operand_t operand) {
  if (operand < 0 || operand >= MFA_OPERAND_COUNT) return "";
  return kOperandNames[operand];
}
int mfa_operand_buffer_binding(mfa_operand_t operand) {
  return (operand >= 0 && operand < MFA_BUFFER_COUNT) ? static_cast<int>(operand) : -1;
}

void mfa_attention_descriptor_init(mfa_attention_descriptor_t *descriptor) {
  if (descriptor) memset(descriptor, 0, sizeof(*descriptor));
}

int mfa_attention_descriptor_memory_precision(const mfa_attention_descriptor_t *descriptor, mfa_operand_t operand,
                                              mfa_precision_t *out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  int p = (operand >= 0 && operand < MFA_OPERAND_COUNT) ? memory_precision(*descriptor, operand) : -1;
  if (p < 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT,
                std::string("Precision of operand ") + mfa_operand_name(operand) + " was not specified.");
  *out = static_cast<mfa_precision_t>(p);
  return MFA_SUCCESS;
}

int mfa_attention_descriptor_register_precision(const mfa_attention_descriptor_t *descriptor, mfa_operand_t operand,
                                                mfa_precision_t *out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  int p = (operand >= 0 && operand < MFA_OPERAND_COUNT) ? register_precision(*descriptor, operand) : -1;
  if (p < 0)
    return fail(MFA_ERROR_INVALID_ARGUMENT,
                std::string("Precision of operand ") + mfa_operand_name(operand) + " was not specified.");
  *out = static_cast<mfa_precision_t>(p);
  return MFA_SUCCESS;
}

void mfa_attention_kernel_descriptor_init(mfa_attention_kernel_descriptor_t *kd) {
  if (!kd) return;
  memset(kd, 0, sizeof(*kd));
  memset(kd->memory_precisions, 0xFF, sizeof(kd->memory_precisions));
  memset(kd->register_precisions, 0xFF, sizeof(kd->register_precisions));
  kd->prefer_async_cache = 0xFF;
  kd->prefer_async_load = 0xFF;
  kd->type = 0xFF;
}

int mfa_attention_kernel_descriptor_get_precision(const mfa_attention_kernel_descriptor_t *kd, mfa_operand_t operand,
                                                  int register_file) {
  if (!kd || operand < 0 || operand >= MFA_OPERAND_COUNT) return -1;
  const uint8_t v = register_file ? kd->register_precisions[operand] : kd->memory_precisions[operand];
  return v == 0xFF ? -1 : static_cast<int>(v);
}

void mfa_attention_kernel_descriptor_set_precision(mfa_attention_kernel_descriptor_t *kd, mfa_operand_t operand,
                                                   int register_file, int value) {
  if (!kd || operand < 0 || operand >= MFA_OPERAND_COUNT) return;
  const uint8_t v = (value < 0 || value > MFA_BF16) ? 0xFF : static_cast<uint8_t>(value);
  (register_file ? kd->register_precisions : kd->memory_precisions)[operand] = v;
}

int mfa_attention_descriptor_kernel_descriptor(const mfa_attention_descriptor_t *descriptor, mfa_kernel_type_t type,
                                               mfa_attention_kernel_descriptor_t *out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  return kernel_descriptor(*descriptor, type, *out);
}

const char *mfa_attention_descriptor_parameter_file(const mfa_attention_descriptor_t *descriptor,
                                                    mfa_kernel_type_t type) {
  if (!descriptor) return "";
  return parameter_file(*descriptor, type);
}

int mfa_set_parameter_table(mfa_kernel_type_t type, int transposed, const char *text) {
  if (type < MFA_FORWARD || type > MFA_BACKWARD_KEY_VALUE) return fail(MFA_ERROR_INVALID_ARGUMENT, "Unrecognized kernel type.");
  const int slot = table_slot(type, transposed != 0);
  if (!text) {
    g_table_overridden[slot] = false;
    g_table_override[slot].clear();
    ++g_table_generation;
    return MFA_SUCCESS;
  }
  // validate before installing: rows parse, operands are the expected ones, tuning values decode
  std::vector<ParameterRow> rows;
  int status = parse_table(text, rows);
  if (status != MFA_SUCCESS) return status;
  if (rows.empty()) return fail(MFA_ERROR_INVALID_ARGUMENT, "Parameter table has no rows.");
  for (const ParameterRow &row : rows) {
    uint16_t v = 0;
    if (!parse_u16(row.parallelization, v) || !parse_u16(row.traversal, v) || !parse_u16(row.head, v))
      return fail(MFA_ERROR_INVALID_ARGUMENT, "Could not decode block dimensions.");
    std::vector<int> operands;
    if ((status = parse_operands(row.cachedOperands, operands)) != MFA_SUCCESS) return status;
    const uint16_t expected = type == MFA_FORWARD ? ((1u << MFA_Q) | (1u << MFA_O))
                              : type == MFA_BACKWARD_QUERY ? ((1u << MFA_Q) | (1u << MFA_dO) | (1u << MFA_dQ))
                                                           : ((1u << MFA_K) | (1u << MFA_V) | (1u << MFA_dV) | (1u << MFA_dK));
    for (int operand : operands)  // createCacheState's check (AttentionDescriptor.swift:69-74), applied to every row
      if (!(expected & (1u << operand)))
        return fail(MFA_ERROR_UNEXPECTED_OPERAND, std::string("Unexpected operand: ") + kOperandNames[operand]);
    if (row.splitMinBlocks.empty()) return fail(MFA_ERROR_INVALID_ARGUMENT, "A tensor-core table row needs the two tuning columns.");
    uint16_t minBlocks = 0, maxSplits = 0;
    if (!parse_u16(row.splitMinBlocks, minBlocks) || !parse_u16(row.splitMax, maxSplits))
      return fail(MFA_ERROR_INVALID_ARGUMENT, "Could not decode tuning columns.");
  }
  g_table_override[slot] = text;
  g_table_overridden[slot] = true;
  ++g_table_generation;
  return MFA_SUCCESS;
}

int mfa_attention_descriptor_set_function_constants(const mfa_attention_descriptor_t *descriptor,
                                                    mfa_function_constants_t *constants) {
  if (!descriptor || !constants) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if (!descriptor->has_matrix_dimensions) return fail(MFA_ERROR_INCOMPLETE_DESCRIPTOR, "Descriptor was incomplete.");
  constants->row = descriptor->row;
  constants->column = descriptor->column;
  constants->batch_count = descriptor->batch_count;
  constants->kv_group = 0;  // the descriptor describes no K/V grouping; the caller sets it
  return MFA_SUCCESS;
}

int mfa_attention_descriptor_operand_elements(const mfa_attention_descriptor_t *descriptor, mfa_operand_t operand,
                                              size_t *out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  if (!descriptor->has_matrix_dimensions) return fail(MFA_ERROR_INCOMPLETE_DESCRIPTOR, "Descriptor was incomplete.");
  const size_t batch = descriptor->batch_count ? descriptor->batch_count : 1;
  size_t n;
  switch (operand) {
    case MFA_Q: case MFA_O: case MFA_dO: case MFA_dQ: n = static_cast<size_t>(descriptor->row) * descriptor->head; break;
    case MFA_K: case MFA_V: case MFA_dK: case MFA_dV: n = static_cast<size_t>(descriptor->column) * descriptor->head; break;
    case MFA_L: case MFA_D: n = descriptor->row; break;
    default: return fail(MFA_ERROR_INVALID_ARGUMENT, "Operand has no buffer.");
  }
  *out = n * batch;
  return MFA_SUCCESS;
}

}  // extern "C"
