// AttentionKernel side of the C ABI: handle creation/validation, launch geometry, and encode()
// -- the compile + bind + dispatch the reference leaves to its caller
// (Tests/FlashAttentionTests/Attention/SquareAttentionTest.swift:240-372).
// Mirrors Sources/FlashAttention/Attention/AttentionKernel/AttentionKernel.swift.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdlib>
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

// Whether the tensor-core family copies this operand into a row-major, pad8(D)-column staging buffer: every operand
// with a head dimension when D % 8 != 0, and any operand stored transposed (L and D are per-row vectors, never staged).
static bool stages_operand(int type, int slot, bool padded, uint16_t transpose_mask) {
  if (slot == MFA_L || slot == MFA_D) return false;
  if (type == MFA_BACKWARD_KEY_VALUE && slot == MFA_O) return false;  // (not read by dK/dV)
  return padded || ((transpose_mask >> slot) & 1);
}

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
  p.exp2_fma_quarters = k->descriptor.exp2_fma_quarters;
  p.split_min_blocks = k->descriptor.split_min_blocks;
  p.split_max = k->descriptor.split_max ? k->descriptor.split_max : 1;
  int n = 0;
  const int *ops = operands_of(k->type, &n);
  for (int i = 0; i < n; ++i)
    if (buffers[ops[i]] == nullptr)
      return fail(MFA_ERROR_INVALID_ARGUMENT, std::string("Buffer ") + mfa_operand_name((mfa_operand_t)ops[i]) +
                                                  " (binding " + std::to_string(ops[i]) + ") is NULL.");
  return MFA_SUCCESS;
}

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
              kd->memory_precisions[MFA_V] == pq &&
              Dp <= (k->type == MFA_FORWARD ? tcgen05_forward_max_head() : tcgen05_backward_max_head());
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
    // tuning columns: every compiled exp2 variant is accepted, anything else is rejected with the list of what exists
    const uint32_t max_quarters = k->type == MFA_FORWARD ? kMaxForwardExp2Quarters : kMaxBackwardExp2Quarters;
    if (kd->exp2_fma_quarters > max_quarters) {
      delete k;
      return fail(MFA_ERROR_UNSUPPORTED, "exp2-on-FMA-pipe fraction " + std::to_string(kd->exp2_fma_quarters) +
                                             "/4 has no compiled sm_90a kernel (available: 0.." +
                                             std::to_string(max_quarters) + ").");
    }
    if (k->type == MFA_FORWARD)
      tcgen05_forward_geometry(Dp, &k->threads, &k->smem_bytes, &k->par, &k->trav, &k->head);
    else
      tcgen05_backward_geometry(k->type, Dp, &k->threads, &k->smem_bytes, &k->par, &k->trav, &k->head);
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
                   ">";
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

int mfa_attention_kernel_grid_size(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                   uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  // parallelization dimension: R for forward / backwardQuery, C for backwardKeyValue
  // (AttentionKernel.swift:197-204; dispatch: SquareAttentionTest.swift:328-339)
  const uint32_t dim = kernel->type == MFA_BACKWARD_KEY_VALUE ? c->column : c->row;
  const uint32_t batch = c->batch_count ? c->batch_count : 1;
  *out = ((dim + kernel->par - 1) / kernel->par) * batch;
  return MFA_SUCCESS;
}

const char *mfa_attention_kernel_source_name(const mfa_attention_kernel_t *kernel) {
  return kernel ? kernel->source_name.c_str() : "";
}

int mfa_attention_kernel_launch_count(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *c,
                                      uint32_t *out) {
  if (!kernel || !c || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  *out = 1;
  if (kernel->backend != MFA_BACKEND_TCGEN05) return MFA_SUCCESS;
  const mfa_attention_kernel_descriptor_t &d = kernel->descriptor;
  const uint32_t Dp = (d.head_dimension + 7u) / 8u * 8u, b = c->batch_count ? c->batch_count : 1;
  if (kernel->type == MFA_FORWARD)
    *out = tcgen05_forward_launch_count(c->row, c->column, Dp, b, d.split_min_blocks, d.split_max);
  else
    *out = tcgen05_backward_launch_count(kernel->type, c->row, c->column, Dp, b, d.split_min_blocks, d.split_max,
                                         d.memory_precisions[MFA_dO] != d.memory_precisions[MFA_Q]);
  // staged operands (head % 8 != 0, or stored transposed): one copy per staged input, one per output
  int n = 0;
  const int *ops = operands_of(kernel->type, &n);
  for (int i = 0; i < n; ++i)
    if (stages_operand(kernel->type, ops[i], d.head_dimension % 8 != 0, d.transpose_state_mask)) *out += 1;
  return MFA_SUCCESS;
}

int mfa_attention_kernel_encode(const mfa_attention_kernel_t *kernel, const mfa_function_constants_t *constants,
                                void *const buffers[MFA_BUFFER_COUNT], void *cuda_stream) {
  if (!kernel || !constants || !buffers) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  int status = check_device();
  if (status != MFA_SUCCESS) return status;
  AttentionParams p;
  status = build_params(kernel, constants, buffers, p);
  if (status != MFA_SUCCESS) return status;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);

  // Several kernels carry the batch in gridDim.y (limit 65535; the SIMT dK/dV kernel multiplies it by up to four head
  // slices): larger batches go out as several launches over slices of the batch -- the problems are independent and
  // stored back to back, so a slice is just a pointer offset.
  constexpr uint32_t kMaxBatchPerLaunch = 16384;
  const uint32_t batch = p.batch;
  size_t head_bytes[kSlots];
  for (int slot = 0; slot < kSlots; ++slot) {
    const size_t seq = (slot == sK || slot == sV || slot == sdK || slot == sdV) ? p.C : p.R;
    const size_t elements = (slot == sL || slot == sD) ? seq : seq * p.D;
    head_bytes[slot] = elements * (p.prec[slot] == FP32 ? 4 : 2);
  }
  // Tensor-core family: operands with D % 8 != 0 or a transposed layout are staged row-major with pad8(D) columns, the
  // kernels run at the padded head dimension (the softmax scale stays 1 / sqrt(D) of the true D), and the FP32 outputs
  // are copied back to the caller's layout without the padding.
  const bool tc = kernel->backend == MFA_BACKEND_TCGEN05;
  const bool padded = tc && p.D % 8 != 0;
  const uint32_t Dp = (p.D + 7) / 8 * 8;
  int n = 0;
  const int *ops = operands_of(kernel->type, &n);
  bool staged = false;
  for (int i = 0; i < n; ++i) staged |= tc && stages_operand(kernel->type, ops[i], padded, kernel->descriptor.transpose_state_mask);
  const int device = staged ? current_device() : 0;
  for (uint32_t h0 = 0; h0 < batch; h0 += kMaxBatchPerLaunch) {
    AttentionParams q = p;
    q.batch = batch - h0 < kMaxBatchPerLaunch ? batch - h0 : kMaxBatchPerLaunch;
    for (int slot = 0; slot < kSlots; ++slot)
      if (q.buf[slot]) q.buf[slot] = static_cast<char *>(q.buf[slot]) + head_bytes[slot] * h0;
    cudaError_t e = cudaSuccess;
    void *user_out[kSlots] = {};  // staged outputs: where the caller's copies go
    if (staged) {
      auto seq_of = [&](int slot) -> uint32_t { return (slot == sK || slot == sV || slot == sdK || slot == sdV) ? p.C : p.R; };
      auto bytes_of = [&](int slot) -> size_t {
        return ((static_cast<size_t>(q.batch) * seq_of(slot) * Dp * (p.prec[slot] == FP32 ? 4 : 2)) + 255) & ~size_t(255);
      };
      size_t total = 0;
      for (int i = 0; i < n; ++i)
        if (stages_operand(kernel->type, ops[i], padded, kernel->descriptor.transpose_state_mask)) total += bytes_of(ops[i]);
      void *ws = nullptr;
      if ((e = workspace_for(device, stream, total, &ws, /*slot=*/1)) != cudaSuccess)
        return fail(MFA_ERROR_CUDA, std::string("staging workspace: ") + cudaGetErrorString(e) + " " + last_launch_detail());
      char *cursor = static_cast<char *>(ws) + kWorkspaceCounterBytes;
      for (int i = 0; i < n && e == cudaSuccess; ++i) {
        const int slot = ops[i];
        if (!stages_operand(kernel->type, slot, padded, kernel->descriptor.transpose_state_mask)) continue;
        if (is_output(kernel->type, slot))
          user_out[slot] = q.buf[slot];
        else
          e = launch_stage_operand(q.buf[slot], cursor, q.batch, seq_of(slot), p.D, Dp, p.prec[slot] == FP32 ? 4 : 2,
                                   q.transposed[slot], stream);
        q.buf[slot] = cursor;
        cursor += bytes_of(slot);
      }
      for (int slot = 0; slot < kSlots; ++slot) q.transposed[slot] = 0;
      q.D = Dp;  // (q.scale / q.scale_log2 keep the true head dimension)
      if (e != cudaSuccess) return fail(MFA_ERROR_CUDA, std::string("operand staging failed: ") + cudaGetErrorString(e));
    }
    if (kernel->backend == MFA_BACKEND_TCGEN05) {
      switch (kernel->type) {
        case MFA_FORWARD: e = launch_tcgen05_forward(q, stream); break;
        case MFA_BACKWARD_QUERY: e = launch_tcgen05_backward_query(q, stream); break;
        default: e = launch_tcgen05_backward_key_value(q, stream); break;
      }
    } else {
      switch (kernel->type) {
        case MFA_FORWARD: e = launch_simt_forward(q, stream); break;
        case MFA_BACKWARD_QUERY: e = launch_simt_backward_query(q, stream); break;
        default: e = launch_simt_backward_key_value(q, stream); break;
      }
    }
    if (e != cudaSuccess)
      return fail(MFA_ERROR_CUDA, std::string("launch of ") + kernel->source_name + " failed: " + cudaGetErrorString(e) +
                                      " " + last_launch_detail());
    if (staged) {
      for (int slot = 0; slot < kSlots && e == cudaSuccess; ++slot)
        if (user_out[slot]) {
          const uint32_t seq = (slot == sdK || slot == sdV) ? p.C : p.R;
          e = launch_unstage_output(static_cast<const float *>(q.buf[slot]), static_cast<float *>(user_out[slot]), q.batch,
                                    seq, p.D, Dp, p.transposed[slot], stream);
        }
      if (e != cudaSuccess) return fail(MFA_ERROR_CUDA, std::string("copy-back of staged outputs failed: ") + cudaGetErrorString(e));
    }
  }
  return MFA_SUCCESS;
}

// Debug-only export (deliberately absent from include/mfa_b200.h): 1 merges split-KV partials inside the attention
// kernel (one launch), 0 (default) in a second launch (tests cover both forms).
MFA_API void mfa_debug_set_forward_fused(int enabled) { tcgen05_forward_set_fused(enabled); }

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
         a.input_precision_override == b.input_precision_override &&
         // with transposed operands the kernel family depends on R % 8 / C % 8 (TMA row pitch)
         select_backend(a, MFA_FORWARD) == select_backend(b, MFA_FORWARD);
}
}  // namespace

int mfa_attention_kernel_cache_fetch(const mfa_attention_descriptor_t *descriptor, mfa_kernel_type_t type,
                                     const mfa_attention_kernel_t **out) {
  if (!descriptor || !out) return fail(MFA_ERROR_INVALID_ARGUMENT, "NULL argument.");
  std::lock_guard<std::mutex> lock(g_cache_mutex);
  for (const auto &entry : g_kernel_cache)
    if (entry.first.type == static_cast<int>(type) && entry.first.table_generation == parameter_table_generation() &&
        same_descriptor(entry.first.descriptor, *descriptor)) {
      *out = entry.second;
      return MFA_SUCCESS;
    }
  mfa_attention_kernel_descriptor_t kd;
  int status = mfa_attention_descriptor_kernel_descriptor(descriptor, type, &kd);
  if (status != MFA_SUCCESS) return status;
  mfa_attention_kernel_t *kernel = nullptr;
  if ((status = mfa_attention_kernel_create(&kd, &kernel)) != MFA_SUCCESS) return status;
  g_kernel_cache.push_back({CacheKey{*descriptor, static_cast<int>(type), parameter_table_generation()}, kernel});
  *out = kernel;
  return MFA_SUCCESS;
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
  // tuning knob (chunk-count sweeps of the host-buffer path): MFA_B200_HOST_CHUNKS=<n>
  if (const char *env = getenv("MFA_B200_HOST_CHUNKS")) {
    const uint32_t n = static_cast<uint32_t>(atoi(env));
    if (n >= 1 && n <= kMaxChunks) return (batch + n - 1) / n;
  }
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
  const char *stats_env = getenv("MFA_B200_HOST_BATCH_STATS");  // tuning knob: 0 = one copy per chunk, as for O
  if (per_chunk < batch && !(stats_env && stats_env[0] == '0'))
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
