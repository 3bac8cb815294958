"""mfa_b200 -- Python mirror of the reference's Swift attention API over the C ABI.

The reference (philipturner/metal-flash-attention) is a Swift package; Swift is not installed in this
image, so the host-side mirror used by tests/ and bench.py is this thin ctypes layer.  It keeps the
reference's names, field meanings and failure behaviour:

    AttentionDescriptor            Sources/FlashAttention/Attention/AttentionDescriptor/AttentionDescriptor.swift:10-27
      .kernelDescriptor(type:)     :33-130
      .setFunctionConstants(_:)    :139-148
      .memoryPrecisions            AttentionDescriptor+Precisions.swift:10-146
      .registerPrecisions          :149-215
    AttentionKernelDescriptor      Attention/AttentionKernelDescriptor.swift:7-48
    AttentionKernelType            Attention/AttentionKernelType.swift:8-23
    AttentionOperand(.bufferBinding)  Attention/AttentionOperand.swift:8-72
    AttentionKernel                Attention/AttentionKernel/AttentionKernel.swift:11-50, 268-363
    GEMMOperandPrecision           GEMM/GEMMOperandPrecision.swift:33-61

All arithmetic happens in libmfa_b200.so (hand-written sm_90a CUDA).  There is no Python or CPU
fallback: if the shared library is missing, importing this package raises.  Where the reference traps
with fatalError(...), this mirror raises MFAError carrying the same message.
"""
from __future__ import annotations

import ctypes
import enum
import os
from typing import Dict, Optional, Sequence, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("MFA_B200_LIBRARY") or os.path.join(_HERE, "lib", "libmfa_b200.so")  # override: tuning builds only

MFA_OPERAND_COUNT = 14
MFA_BUFFER_COUNT = 10


class MFAError(RuntimeError):
    """Raised where the reference would fatalError(); .status is the mfa_status_t code."""

    def __init__(self, status: int, message: str):
        super().__init__(f"[mfa status {status}] {message}")
        self.status = status
        self.message = message


# -------------------------------------------------------------------------------------------------
# C structs (must match include/mfa_b200.h)
# -------------------------------------------------------------------------------------------------
class _CDescriptor(ctypes.Structure):
    _fields_ = [
        ("low_precision_inputs", ctypes.c_uint8),
        ("low_precision_intermediates", ctypes.c_uint8),
        ("has_matrix_dimensions", ctypes.c_uint8),
        ("has_transpose_state", ctypes.c_uint8),
        ("row", ctypes.c_uint32),
        ("column", ctypes.c_uint32),
        ("head", ctypes.c_uint16),
        ("transpose_Q", ctypes.c_uint8),
        ("transpose_K", ctypes.c_uint8),
        ("transpose_V", ctypes.c_uint8),
        ("transpose_O", ctypes.c_uint8),
        ("input_precision_override", ctypes.c_uint8),
        ("causal", ctypes.c_uint8),
        ("batch_count", ctypes.c_uint32),
    ]


class _CKernelDescriptor(ctypes.Structure):
    _fields_ = [
        ("has_block_dimensions", ctypes.c_uint8),
        ("block_parallelization", ctypes.c_uint16),
        ("block_traversal", ctypes.c_uint16),
        ("block_head", ctypes.c_uint16),
        ("cache_state_valid_mask", ctypes.c_uint16),
        ("cache_state_mask", ctypes.c_uint16),
        ("has_head_dimension", ctypes.c_uint8),
        ("head_dimension", ctypes.c_uint16),
        ("memory_precisions", ctypes.c_uint8 * MFA_OPERAND_COUNT),
        ("register_precisions", ctypes.c_uint8 * MFA_OPERAND_COUNT),
        ("prefer_async_cache", ctypes.c_uint8),
        ("prefer_async_load", ctypes.c_uint8),
        ("transpose_state_valid_mask", ctypes.c_uint16),
        ("transpose_state_mask", ctypes.c_uint16),
        ("type", ctypes.c_uint8),
        ("backend", ctypes.c_uint8),
        ("split_min_blocks", ctypes.c_uint8),
        ("split_max", ctypes.c_uint8),
        ("causal", ctypes.c_uint8),
    ]


class _CFunctionConstants(ctypes.Structure):
    _fields_ = [("row", ctypes.c_uint32), ("column", ctypes.c_uint32), ("batch_count", ctypes.c_uint32),
                ("kv_group", ctypes.c_uint32)]


class SequenceTable(ctypes.Structure):
    """mfa_sequence_table_t: packed variable-length sequences (FlashAttention's cu_seqlens).  Sequence s owns query rows
    [row_offsets[s], row_offsets[s + 1]) and key rows [column_offsets[s], column_offsets[s + 1]) of every problem; the
    offsets are int32 DEVICE pointers with count + 1 entries, max_row / max_column bound every sequence's lengths."""
    _fields_ = [("count", ctypes.c_uint32), ("max_row", ctypes.c_uint32), ("max_column", ctypes.c_uint32),
                ("row_offsets", ctypes.c_void_p), ("column_offsets", ctypes.c_void_p)]

    def __init__(self, count=0, max_row=0, max_column=0, row_offsets=0, column_offsets=0):
        super().__init__(int(count), int(max_row), int(max_column), row_offsets or None, column_offsets or None)


class PagedKV(ctypes.Structure):
    """mfa_paged_kv_t: the forward over packed queries (row_offsets, as in SequenceTable) whose keys and values live in
    page pools [num_pages][page_size][Hkv][D] (vLLM's block table).  Sequence s has column_lengths[s] keys, key i in pool
    row page_table[s * page_stride + i // page_size] * page_size + i % page_size.  The three tables are int32 DEVICE
    pointers; max_row bounds every sequence's query count."""
    _fields_ = [("count", ctypes.c_uint32), ("max_row", ctypes.c_uint32), ("row_offsets", ctypes.c_void_p),
                ("column_lengths", ctypes.c_void_p), ("page_table", ctypes.c_void_p), ("page_stride", ctypes.c_uint32),
                ("page_size", ctypes.c_uint32)]

    def __init__(self, count=0, max_row=0, row_offsets=0, column_lengths=0, page_table=0, page_stride=0,
                 page_size=0):
        super().__init__(int(count), int(max_row), row_offsets or None, column_lengths or None, page_table or None,
                         int(page_stride), int(page_size))


class SplitKV(ctypes.Structure):
    """mfa_split_kv_t: a split-KV forward over packed sequences or a paged cache (FlashAttention's num_splits).
    num_splits 0 lets the library plan; 1..16 is taken as given.  max_column: a planning hint bounding every
    sequence's keys (0 = the table's bound), never a correctness contract."""
    _fields_ = [("num_splits", ctypes.c_uint32), ("max_column", ctypes.c_uint32)]

    def __init__(self, num_splits=0, max_column=0):
        super().__init__(int(num_splits), int(max_column))


class SplitPlan(ctypes.Structure):
    """mfa_split_plan_t: key ranges per tile, query heads per tile, CTAs of the attention kernel, kernels launched."""
    _fields_ = [("splits", ctypes.c_uint32), ("heads_per_tile", ctypes.c_uint32), ("grid_size", ctypes.c_uint32),
                ("launch_count", ctypes.c_uint32)]


class FP8KV(ctypes.Structure):
    """mfa_fp8_kv_t: the K and V pools of a paged call hold FP8 E4M3 bytes (torch.float8_e4m3fn viewed as uint8), key
    row i of K/V head kv standing for k_scale[kv] * e4m3(byte) (v_scale for V).  k_scale / v_scale: float32 DEVICE
    pointers with one entry per K/V head, read at launch; 0 means every scale is 1."""
    _fields_ = [("k_scale", ctypes.c_void_p), ("v_scale", ctypes.c_void_p)]

    def __init__(self, k_scale=0, v_scale=0):
        super().__init__(k_scale or None, v_scale or None)


class PagedKVAppend(ctypes.Structure):
    """mfa_paged_kv_append_t: the step's new tokens for appendPagedKV.  k_new / v_new: DEVICE pointers, token t's K/V
    head kv at element t * token_stride + kv * head_dimension (token_stride 0: kv_heads * head_dimension, a contiguous
    [rows][kv_heads][head_dimension] tensor); rows: tokens they hold; pool_rows: rows of each pool (num_pages *
    page_size); precision: a GEMMOperandPrecision of k_new / v_new."""
    _fields_ = [("k_new", ctypes.c_void_p), ("v_new", ctypes.c_void_p), ("rows", ctypes.c_uint32),
                ("token_stride", ctypes.c_uint32), ("kv_heads", ctypes.c_uint32), ("head_dimension", ctypes.c_uint32),
                ("pool_rows", ctypes.c_uint32), ("precision", ctypes.c_uint32)]

    def __init__(self, k_new=0, v_new=0, rows=0, token_stride=0, kv_heads=0, head_dimension=0, pool_rows=0,
                 precision=0):
        super().__init__(k_new or None, v_new or None, int(rows), int(token_stride), int(kv_heads), int(head_dimension),
                         int(pool_rows), int(precision))


class Rotary(ctypes.Structure):
    """mfa_rotary_t: rotary position embedding for appendPagedKV(..., rotary=).  q_new: DEVICE pointer, token t's query
    head h at element t * q_token_stride + h * D (0: query_heads * D, a contiguous [rows][query_heads][D] tensor), in
    append.precision; q_out: the paged forward's Q buffer [query_heads][append.rows][D]; cos / sin: float32 DEVICE
    tables, position p, frequency j < rotary_dim / 2 at p * table_stride + j (0: rotary_dim / 2); positions: their
    rows, at least page_stride * page_size; interleaved: 0 pairs (j, j + r/2) (GPT-NeoX / Llama), 1 pairs (2j, 2j + 1)
    (GPT-J)."""
    _fields_ = [("q_new", ctypes.c_void_p), ("q_out", ctypes.c_void_p), ("cos", ctypes.c_void_p),
                ("sin", ctypes.c_void_p), ("query_heads", ctypes.c_uint32), ("q_token_stride", ctypes.c_uint32),
                ("rotary_dim", ctypes.c_uint32), ("table_stride", ctypes.c_uint32), ("positions", ctypes.c_uint32),
                ("interleaved", ctypes.c_uint32)]

    def __init__(self, q_new=0, q_out=0, cos=0, sin=0, query_heads=0, q_token_stride=0, rotary_dim=0, table_stride=0,
                 positions=0, interleaved=0):
        super().__init__(q_new or None, q_out or None, cos or None, sin or None, int(query_heads), int(q_token_stride),
                         int(rotary_dim), int(table_stride), int(positions), int(interleaved))


class _CWindow(ctypes.Structure):
    _fields_ = [("left", ctypes.c_int32), ("right", ctypes.c_int32)]


def _window(window) -> "_CWindow":
    left, right = (int(v) for v in window)
    for name, v in (("left", left), ("right", right)):
        if not -2**31 <= v < 2**31:   # (ctypes would wrap it; values in int32 are checked by the library)
            raise MFAError(-2, f"Window: {name} {v} is outside [-1, {2**31 - 1}].")
    return _CWindow(left, right)


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is deliberately no Python/CPU fallback for the attention kernels)")
    lib = ctypes.CDLL(_LIB_PATH)
    c = ctypes
    lib.mfa_last_error.restype = c.c_char_p
    lib.mfa_version.restype = c.c_char_p
    lib.mfa_precision_name.restype = c.c_char_p
    lib.mfa_operand_name.restype = c.c_char_p
    lib.mfa_attention_kernel_source_name.restype = c.c_char_p
    lib.mfa_attention_kernel_source_name.argtypes = [c.c_void_p]
    lib.mfa_attention_descriptor_parameter_file.restype = c.c_char_p
    lib.mfa_attention_descriptor_parameter_file.argtypes = [c.POINTER(_CDescriptor), c.c_int]
    lib.mfa_attention_descriptor_memory_precision.argtypes = [c.POINTER(_CDescriptor), c.c_int, c.POINTER(c.c_int)]
    lib.mfa_attention_descriptor_register_precision.argtypes = [c.POINTER(_CDescriptor), c.c_int, c.POINTER(c.c_int)]
    lib.mfa_attention_descriptor_kernel_descriptor.argtypes = [c.POINTER(_CDescriptor), c.c_int,
                                                               c.POINTER(_CKernelDescriptor)]
    lib.mfa_attention_descriptor_set_function_constants.argtypes = [c.POINTER(_CDescriptor),
                                                                    c.POINTER(_CFunctionConstants)]
    lib.mfa_attention_descriptor_operand_elements.argtypes = [c.POINTER(_CDescriptor), c.c_int,
                                                              c.POINTER(c.c_size_t)]
    lib.mfa_attention_kernel_descriptor_init.argtypes = [c.POINTER(_CKernelDescriptor)]
    lib.mfa_attention_kernel_create.argtypes = [c.POINTER(_CKernelDescriptor), c.POINTER(c.c_void_p)]
    lib.mfa_attention_kernel_destroy.argtypes = [c.c_void_p]
    lib.mfa_attention_kernel_destroy.restype = None
    lib.mfa_attention_kernel_block_dimensions.argtypes = [c.c_void_p, c.POINTER(c.c_uint16 * 3)]
    lib.mfa_attention_kernel_threadgroup_size.argtypes = [c.c_void_p, c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_threadgroup_memory_allocation.argtypes = [c.c_void_p, c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_grid_size.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants), c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_launch_count.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                      c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_encode.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_void_p]
    lib.mfa_attention_kernel_encode_sequences.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                          c.POINTER(SequenceTable),
                                                          c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_void_p]
    lib.mfa_attention_kernel_grid_size_sequences.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                             c.POINTER(SequenceTable), c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_launch_count_sequences.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                                c.POINTER(SequenceTable), c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_encode_paged.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants), c.POINTER(PagedKV),
                                                      c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_void_p]
    lib.mfa_attention_kernel_grid_size_paged.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                         c.POINTER(PagedKV), c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_launch_count_paged.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                            c.POINTER(PagedKV), c.POINTER(c.c_uint32)]
    lib.mfa_attention_kernel_encode_sequences_split.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                                c.POINTER(SequenceTable), c.POINTER(SplitKV),
                                                                c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_void_p]
    lib.mfa_attention_kernel_encode_paged_split.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                            c.POINTER(PagedKV), c.POINTER(SplitKV),
                                                            c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_void_p]
    lib.mfa_attention_kernel_encode_paged_fp8.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                          c.POINTER(PagedKV), c.POINTER(SplitKV), c.POINTER(FP8KV),
                                                          c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_void_p]
    lib.mfa_attention_kernel_split_plan.argtypes = [c.c_void_p, c.POINTER(_CFunctionConstants),
                                                    c.POINTER(SequenceTable), c.POINTER(PagedKV), c.POINTER(SplitKV),
                                                    c.POINTER(SplitPlan)]
    lib.mfa_paged_kv_append.argtypes = [c.POINTER(PagedKV), c.POINTER(PagedKVAppend), c.c_void_p, c.c_void_p,
                                        c.POINTER(FP8KV), c.c_void_p]
    lib.mfa_paged_kv_append_rotary.argtypes = [c.POINTER(PagedKV), c.POINTER(PagedKVAppend), c.POINTER(Rotary),
                                               c.c_void_p, c.c_void_p, c.POINTER(FP8KV), c.c_void_p]
    lib.mfa_attention_kernel_cache_fetch.argtypes = [c.POINTER(_CDescriptor), c.c_int, c.POINTER(c.c_void_p)]
    lib.mfa_attention_kernel_create_windowed.argtypes = [c.POINTER(_CKernelDescriptor), c.POINTER(_CWindow),
                                                         c.POINTER(c.c_void_p)]
    lib.mfa_attention_kernel_cache_fetch_windowed.argtypes = [c.POINTER(_CDescriptor), c.c_int, c.POINTER(_CWindow),
                                                              c.POINTER(c.c_void_p)]
    lib.mfa_attention_kernel_cache_size.restype = c.c_int
    lib.mfa_attention_run_host.argtypes = [c.POINTER(_CDescriptor), c.c_uint32,
                                           c.POINTER(c.c_void_p * MFA_BUFFER_COUNT), c.c_int]
    try:
        lib.mfa_set_parameter_table.argtypes = [c.c_int, c.c_int, c.c_char_p]
        lib.mfa_host_alloc.argtypes = [c.c_size_t, c.c_int, c.POINTER(c.c_void_p)]
        lib.mfa_host_alloc_upload.argtypes = [c.c_size_t, c.c_int, c.POINTER(c.c_void_p)]
        lib.mfa_host_free.argtypes = [c.c_void_p]
        lib.mfa_host_bind_thread_to_device.argtypes = [c.c_int, c.POINTER(c.c_int)]
        lib.mfa_release_device_resources.argtypes = [c.c_int]
    except AttributeError:
        # only an older tuning build selected through MFA_B200_LIBRARY can lack these (A/B timing against it still works)
        if not os.environ.get("MFA_B200_LIBRARY"):
            raise
    return lib


_lib = _load()


def _check(status: int):
    if status != 0:
        raise MFAError(status, _lib.mfa_last_error().decode())


def hostAlloc(nbytes: int, device: int = 0, upload: bool = False) -> int:
    """mfa_host_alloc: page-locked host buffer on the NUMA node of `device` (for runHost); returns the address.
    upload=True (mfa_host_alloc_upload): write-combined pages for buffers the host only writes (Q, K, V, dO)."""
    out = ctypes.c_void_p()
    _check((_lib.mfa_host_alloc_upload if upload else _lib.mfa_host_alloc)(int(nbytes), int(device), ctypes.byref(out)))
    return out.value


def hostFree(address: int) -> None:
    _check(_lib.mfa_host_free(ctypes.c_void_p(address)))


def bindThreadToDevice(device: int = 0) -> int:
    """mfa_host_bind_thread_to_device: pin the calling thread to the CPUs of the GPU's NUMA node; returns the node
    (-1: the platform reports none, nothing changed)."""
    node = ctypes.c_int(-1)
    _check(_lib.mfa_host_bind_thread_to_device(int(device), ctypes.byref(node)))
    return node.value


def releaseDeviceResources(device: int = 0) -> None:
    """mfa_release_device_resources: free the library's scratch and workspaces on `device`."""
    _check(_lib.mfa_release_device_resources(int(device)))


def setParameterTable(type: "AttentionKernelType", text: Optional[str], transposed: bool = False) -> None:
    """mfa_set_parameter_table: replace (text) or restore (None) the tensor-core-family parameter table of `type`."""
    _check(_lib.mfa_set_parameter_table(int(type), int(bool(transposed)),
                                        None if text is None else text.encode()))


def appendPagedKV(paged: PagedKV, append: PagedKVAppend, k_pool: int, v_pool: int, fp8: Optional[FP8KV] = None,
                  stream: int = 0, rotary: Optional[Rotary] = None) -> None:
    """mfa_paged_kv_append: writes the step's new keys and values into the page pools k_pool / v_pool (DEVICE pointers)
    through the table of the step's paged forward.  New token i of sequence s becomes key column_lengths[s] - Rs + i.
    fp8: the pools hold E4M3 bytes, each value divided by its K/V head's scale and saturated to +-448; None: the pools
    hold append.precision elements, copied bit for bit.  One launch on `stream` (a cudaStream_t as int), capturable
    into a CUDA graph.
    rotary (mfa_paged_kv_append_rotary): the queries and new keys are also rotated by RoPE at their cache positions,
    and the queries written to rotary.q_out in the paged forward's [query_heads][rows][D] layout, in the same launch."""
    args = (ctypes.byref(paged) if paged is not None else None, ctypes.byref(append) if append is not None else None)
    tail = (ctypes.c_void_p(k_pool or None), ctypes.c_void_p(v_pool or None),
            ctypes.byref(fp8) if fp8 is not None else None, ctypes.c_void_p(stream))
    if rotary is None:
        _check(_lib.mfa_paged_kv_append(*args, *tail))
    else:
        _check(_lib.mfa_paged_kv_append_rotary(*args, ctypes.byref(rotary), *tail))


def library_path() -> str:
    return _LIB_PATH


def version() -> str:
    return _lib.mfa_version().decode()


# -------------------------------------------------------------------------------------------------
# Enumerations
# -------------------------------------------------------------------------------------------------
class GEMMOperandPrecision(enum.IntEnum):
    """GEMMOperandPrecision.swift:33-61 (raw values are ABI)."""
    FP32 = 0
    FP16 = 1
    BF16 = 2

    @property
    def size(self) -> int:
        return 4 if self == GEMMOperandPrecision.FP32 else 2


class AttentionKernelType(enum.IntEnum):
    """AttentionKernelType.swift:8-23."""
    forward = 0
    backwardQuery = 1
    backwardKeyValue = 2


class AttentionOperand(enum.IntEnum):
    """AttentionOperand.swift:8-72; values 0..9 are the buffer bindings."""
    Q = 0
    K = 1
    V = 2
    O = 3
    L = 4
    D = 5
    dO = 6
    dV = 7
    dK = 8
    dQ = 9
    S = 10
    P = 11
    dP = 12
    dS = 13

    @property
    def bufferBinding(self) -> Optional[int]:
        return int(self) if int(self) < MFA_BUFFER_COUNT else None

    @property
    def description(self) -> str:
        return self.name


class Backend(enum.IntEnum):
    simtFP32 = 0
    tcgen05 = 1


# -------------------------------------------------------------------------------------------------
# AttentionDescriptor
# -------------------------------------------------------------------------------------------------
class AttentionDescriptor:
    """AttentionDescriptor.swift:10-27.  `matrixDimensions = (row, column, head)`,
    `transposeState = (Q, K, V, O)`; both start as None (Swift optionals)."""

    def __init__(self):
        self.lowPrecisionInputs: bool = False
        self.lowPrecisionIntermediates: bool = False
        self.matrixDimensions: Optional[Tuple[int, int, int]] = None
        self.transposeState: Optional[Tuple[bool, bool, bool, bool]] = None
        # library extensions (include/mfa_b200.h): None = reference policy (FP16 inputs).
        self.inputPrecisionOverride: Optional[GEMMOperandPrecision] = None
        self.batchCount: int = 1
        # causal mask aligned bottom-right: query row i sees key j iff j <= i + (column - row); rows with no visible key
        # (row > column) get O = 0, L = +inf, D = 0, dQ = 0
        self.causal: bool = False

    def _c(self) -> _CDescriptor:
        d = _CDescriptor()
        d.low_precision_inputs = int(bool(self.lowPrecisionInputs))
        d.low_precision_intermediates = int(bool(self.lowPrecisionIntermediates))
        if self.matrixDimensions is not None:
            d.has_matrix_dimensions = 1
            d.row, d.column, d.head = (int(x) for x in self.matrixDimensions)
        if self.transposeState is not None:
            d.has_transpose_state = 1
            d.transpose_Q, d.transpose_K, d.transpose_V, d.transpose_O = (int(bool(x)) for x in self.transposeState)
        d.input_precision_override = int(self.inputPrecisionOverride) if self.inputPrecisionOverride else 0
        d.batch_count = int(self.batchCount)
        d.causal = int(self.causal)  # (any value other than 0 / 1 is passed on, and rejected by the library)
        return d

    @property
    def memoryPrecisions(self) -> Dict[AttentionOperand, GEMMOperandPrecision]:
        c, out = self._c(), {}
        for op in list(AttentionOperand)[:MFA_BUFFER_COUNT]:
            value = ctypes.c_int()
            _check(_lib.mfa_attention_descriptor_memory_precision(ctypes.byref(c), int(op), ctypes.byref(value)))
            out[op] = GEMMOperandPrecision(value.value)
        return out

    @property
    def registerPrecisions(self) -> Dict[AttentionOperand, GEMMOperandPrecision]:
        c, out = self._c(), {}
        for op in AttentionOperand:
            value = ctypes.c_int()
            _check(_lib.mfa_attention_descriptor_register_precision(ctypes.byref(c), int(op), ctypes.byref(value)))
            out[op] = GEMMOperandPrecision(value.value)
        return out

    def parameterFile(self, type: AttentionKernelType) -> str:
        c = self._c()
        return _lib.mfa_attention_descriptor_parameter_file(ctypes.byref(c), int(type)).decode()

    def kernelDescriptor(self, type: AttentionKernelType) -> "AttentionKernelDescriptor":
        c = self._c()
        out = AttentionKernelDescriptor()
        _check(_lib.mfa_attention_descriptor_kernel_descriptor(ctypes.byref(c), int(type), ctypes.byref(out._c)))
        return out

    def setFunctionConstants(self, constants: "FunctionConstantValues") -> None:
        c = self._c()
        _check(_lib.mfa_attention_descriptor_set_function_constants(ctypes.byref(c), ctypes.byref(constants._c)))

    def operandElements(self, operand: AttentionOperand) -> int:
        c, n = self._c(), ctypes.c_size_t()
        _check(_lib.mfa_attention_descriptor_operand_elements(ctypes.byref(c), int(operand), ctypes.byref(n)))
        return n.value

    def runHost(self, types: Sequence[AttentionKernelType], hostBuffers: Dict[AttentionOperand, int],
                device: int = 0) -> None:
        """End-to-end call on HOST pointers (mfa_attention_run_host): H2D -> kernels -> D2H."""
        c = self._c()
        mask = 0
        for t in types:
            mask |= 1 << int(t)
        arr = (ctypes.c_void_p * MFA_BUFFER_COUNT)()
        for op, ptr in hostBuffers.items():
            arr[int(op)] = ptr
        _check(_lib.mfa_attention_run_host(ctypes.byref(c), mask, ctypes.byref(arr), device))


class FunctionConstantValues:
    """Stand-in for MTLFunctionConstantValues: R at index 0, C at index 1 (AttentionDescriptor.swift:144-147)."""

    def __init__(self):
        self._c = _CFunctionConstants()

    @property
    def row(self) -> int:
        return self._c.row

    @property
    def column(self) -> int:
        return self._c.column

    @property
    def batchCount(self) -> int:
        return self._c.batch_count

    # ---- library extension: grouped-query / multi-query attention
    @property
    def kvGroup(self) -> int:
        """Query problems per K/V problem (0 or 1: every problem has its own K and V).  Query problem b reads K/V
        problem b // kvGroup; K, V, dK, dV hold batchCount // kvGroup problems and dK / dV are summed per group.
        For [B, Hq, N, D] queries and [B, Hkv, N, D] keys: batchCount = B * Hq, kvGroup = Hq // Hkv.
        setFunctionConstants writes 0; set this afterwards."""
        return self._c.kv_group

    @kvGroup.setter
    def kvGroup(self, value: int) -> None:
        self._c.kv_group = int(value)


# -------------------------------------------------------------------------------------------------
# AttentionKernelDescriptor
# -------------------------------------------------------------------------------------------------
class AttentionKernelDescriptor:
    """AttentionKernelDescriptor.swift:7-48 (a plain, editable value)."""

    def __init__(self):
        self._c = _CKernelDescriptor()
        _lib.mfa_attention_kernel_descriptor_init(ctypes.byref(self._c))

    @property
    def blockDimensions(self) -> Optional[Tuple[int, int, int]]:
        if not self._c.has_block_dimensions:
            return None
        return (self._c.block_parallelization, self._c.block_traversal, self._c.block_head)

    @blockDimensions.setter
    def blockDimensions(self, value):
        if value is None:
            self._c.has_block_dimensions = 0
        else:
            self._c.has_block_dimensions = 1
            self._c.block_parallelization, self._c.block_traversal, self._c.block_head = (int(v) for v in value)

    @property
    def cacheState(self) -> Dict[AttentionOperand, bool]:
        return {op: bool((self._c.cache_state_mask >> int(op)) & 1) for op in AttentionOperand
                if (self._c.cache_state_valid_mask >> int(op)) & 1}

    @property
    def headDimension(self) -> Optional[int]:
        return self._c.head_dimension if self._c.has_head_dimension else None

    @headDimension.setter
    def headDimension(self, value):
        self._c.has_head_dimension = 0 if value is None else 1
        self._c.head_dimension = 0 if value is None else int(value)

    def _precisions(self, array) -> Dict[AttentionOperand, GEMMOperandPrecision]:
        return {op: GEMMOperandPrecision(array[int(op)]) for op in AttentionOperand if array[int(op)] != 0xFF}

    @property
    def memoryPrecisions(self):
        return self._precisions(self._c.memory_precisions)

    @property
    def registerPrecisions(self):
        return self._precisions(self._c.register_precisions)

    def setMemoryPrecision(self, operand: AttentionOperand, precision: Optional[GEMMOperandPrecision]):
        self._c.memory_precisions[int(operand)] = 0xFF if precision is None else int(precision)

    def setRegisterPrecision(self, operand: AttentionOperand, precision: Optional[GEMMOperandPrecision]):
        self._c.register_precisions[int(operand)] = 0xFF if precision is None else int(precision)

    @property
    def preferAsyncCache(self) -> Optional[bool]:
        return None if self._c.prefer_async_cache == 0xFF else bool(self._c.prefer_async_cache)

    @preferAsyncCache.setter
    def preferAsyncCache(self, value):
        self._c.prefer_async_cache = 0xFF if value is None else int(bool(value))

    @property
    def preferAsyncLoad(self) -> Optional[bool]:
        return None if self._c.prefer_async_load == 0xFF else bool(self._c.prefer_async_load)

    @preferAsyncLoad.setter
    def preferAsyncLoad(self, value):
        self._c.prefer_async_load = 0xFF if value is None else int(bool(value))

    @property
    def transposeState(self) -> Dict[AttentionOperand, bool]:
        return {op: bool((self._c.transpose_state_mask >> int(op)) & 1) for op in AttentionOperand
                if (self._c.transpose_state_valid_mask >> int(op)) & 1}

    @property
    def type(self) -> Optional[AttentionKernelType]:
        return None if self._c.type == 0xFF else AttentionKernelType(self._c.type)

    @type.setter
    def type(self, value):
        self._c.type = 0xFF if value is None else int(value)

    @property
    def backend(self) -> Backend:
        return Backend(self._c.backend)

    @backend.setter
    def backend(self, value):
        self._c.backend = int(value)

    # ---- library extension: the tuning columns of the parameter-table row (plain, editable data like blockDimensions)
    @property
    def splitPolicy(self) -> Tuple[int, int]:
        """(minimum blocks per traversal range, maximum ranges) for small grids; minimum 0 = never split."""
        return (self._c.split_min_blocks, self._c.split_max)

    @splitPolicy.setter
    def splitPolicy(self, value):
        self._c.split_min_blocks, self._c.split_max = (int(v) for v in value)

    # ---- library extension: the causal mask (AttentionDescriptor.causal), editable like the fields above
    @property
    def causal(self) -> bool:
        return bool(self._c.causal)

    @causal.setter
    def causal(self, value):
        self._c.causal = int(value)


# -------------------------------------------------------------------------------------------------
# AttentionKernel
# -------------------------------------------------------------------------------------------------
def _one_table(sequences, paged):
    if sequences is not None and paged is not None:
        raise MFAError(-2, "Pass sequences= or paged=, not both: a paged call carries its own query offsets.")


class AttentionKernel:
    """AttentionKernel.swift:11-50.  `encode` performs what the reference's callers do by hand
    (makeLibrary / makeComputePipelineState / setBuffer x10 / dispatchThreadgroups,
    SquareAttentionTest.swift:240-372) against DEVICE pointers."""

    def __init__(self, descriptor: AttentionKernelDescriptor, window: Optional[Tuple[int, int]] = None):
        """window: a sliding window (left, right) (mfa_attention_kernel_create_windowed): with delta = column - row,
        query row i sees key j iff i + delta - left <= j <= i + delta + right, -1 leaving a side unbounded.  A causal
        kernel takes right = 0 or -1; (W - 1, 0) is a window of W keys ending at the diagonal."""
        self._handle = ctypes.c_void_p()
        self._owned = True
        if window is None:
            _check(_lib.mfa_attention_kernel_create(ctypes.byref(descriptor._c), ctypes.byref(self._handle)))
        else:
            w = _window(window)
            _check(_lib.mfa_attention_kernel_create_windowed(ctypes.byref(descriptor._c), ctypes.byref(w),
                                                             ctypes.byref(self._handle)))

    @classmethod
    def cached(cls, descriptor: AttentionDescriptor, type: AttentionKernelType,
               window: Optional[Tuple[int, int]] = None) -> "AttentionKernel":
        """mfa_attention_kernel_cache_fetch: the kernel object for (descriptor, type), built once per process and
        owned by the library (the analogue of GEMMKernel.pipelineCache, GEMMDescriptor+PipelineCache.swift:16-36).
        window: a sliding window as in __init__ (mfa_attention_kernel_cache_fetch_windowed, keyed by the window too)."""
        self = cls.__new__(cls)
        self._handle = ctypes.c_void_p()
        self._owned = False
        c = descriptor._c()
        if window is None:
            _check(_lib.mfa_attention_kernel_cache_fetch(ctypes.byref(c), int(type), ctypes.byref(self._handle)))
        else:
            w = _window(window)
            _check(_lib.mfa_attention_kernel_cache_fetch_windowed(ctypes.byref(c), int(type), ctypes.byref(w),
                                                                  ctypes.byref(self._handle)))
        return self

    @staticmethod
    def cacheSize() -> int:
        return _lib.mfa_attention_kernel_cache_size()

    def __del__(self):
        handle = getattr(self, "_handle", None)
        if handle and getattr(self, "_owned", False) and _lib is not None:  # _lib is None during interpreter teardown
            _lib.mfa_attention_kernel_destroy(handle)
            self._handle = None

    @property
    def blockDimensions(self) -> Tuple[int, int, int]:
        out = (ctypes.c_uint16 * 3)()
        _check(_lib.mfa_attention_kernel_block_dimensions(self._handle, ctypes.byref(out)))
        return (out[0], out[1], out[2])

    @property
    def threadgroupSize(self) -> int:
        out = ctypes.c_uint32()
        _check(_lib.mfa_attention_kernel_threadgroup_size(self._handle, ctypes.byref(out)))
        return out.value

    @property
    def threadgroupMemoryAllocation(self) -> int:
        out = ctypes.c_uint32()
        _check(_lib.mfa_attention_kernel_threadgroup_memory_allocation(self._handle, ctypes.byref(out)))
        return out.value

    def gridSize(self, constants: FunctionConstantValues, sequences: Optional[SequenceTable] = None,
                 paged: Optional[PagedKV] = None) -> int:
        """sequences: packed variable-length sequences (mfa_attention_kernel_grid_size_sequences); paged: a paged K/V
        cache (mfa_attention_kernel_grid_size_paged)."""
        out = ctypes.c_uint32()
        _one_table(sequences, paged)
        if paged is not None:
            _check(_lib.mfa_attention_kernel_grid_size_paged(self._handle, ctypes.byref(constants._c),
                                                             ctypes.byref(paged), ctypes.byref(out)))
        elif sequences is None:
            _check(_lib.mfa_attention_kernel_grid_size(self._handle, ctypes.byref(constants._c), ctypes.byref(out)))
        else:
            _check(_lib.mfa_attention_kernel_grid_size_sequences(self._handle, ctypes.byref(constants._c),
                                                                 ctypes.byref(sequences), ctypes.byref(out)))
        return out.value

    def launchCount(self, constants: FunctionConstantValues, sequences: Optional[SequenceTable] = None,
                    paged: Optional[PagedKV] = None) -> int:
        out = ctypes.c_uint32()
        _one_table(sequences, paged)
        if paged is not None:
            _check(_lib.mfa_attention_kernel_launch_count_paged(self._handle, ctypes.byref(constants._c),
                                                                ctypes.byref(paged), ctypes.byref(out)))
        elif sequences is None:
            _check(_lib.mfa_attention_kernel_launch_count(self._handle, ctypes.byref(constants._c), ctypes.byref(out)))
        else:
            _check(_lib.mfa_attention_kernel_launch_count_sequences(self._handle, ctypes.byref(constants._c),
                                                                    ctypes.byref(sequences), ctypes.byref(out)))
        return out.value

    def sourceName(self) -> str:
        """Stands in for createSource() (AttentionKernel+Source.swift:11-55): the kernels are AOT-compiled."""
        return _lib.mfa_attention_kernel_source_name(self._handle).decode()

    def splitPlan(self, constants: FunctionConstantValues, sequences: Optional[SequenceTable] = None,
                  paged: Optional[PagedKV] = None, split: Optional[SplitKV] = None) -> SplitPlan:
        """mfa_attention_kernel_split_plan: what encode(..., split=split) with this table launches.  Exactly one of
        sequences / paged."""
        out = SplitPlan()
        _check(_lib.mfa_attention_kernel_split_plan(self._handle, ctypes.byref(constants._c),
                                                    ctypes.byref(sequences) if sequences is not None else None,
                                                    ctypes.byref(paged) if paged is not None else None,
                                                    ctypes.byref(split) if split is not None else None,
                                                    ctypes.byref(out)))
        return out

    def encode(self, constants: FunctionConstantValues, buffers: Dict[AttentionOperand, int],
               stream: int = 0, sequences: Optional[SequenceTable] = None, paged: Optional[PagedKV] = None,
               split: Optional[SplitKV] = None, fp8: Optional[FP8KV] = None) -> None:
        """buffers: {AttentionOperand: device pointer}; stream: cudaStream_t as int (0 = default).  sequences: packed
        variable-length sequences over the rows of every problem (mfa_attention_kernel_encode_sequences).  paged: the
        forward over a paged K/V cache, K and V pointing at the page pools (mfa_attention_kernel_encode_paged).
        split: the split-KV forward over sequences= or paged= (mfa_attention_kernel_encode_sequences_split / _paged_split).
        fp8: the pools of paged= hold FP8 E4M3 bytes with per-K/V-head scales, with or without split=
        (mfa_attention_kernel_encode_paged_fp8)."""
        _one_table(sequences, paged)
        if split is not None and sequences is None and paged is None:
            raise MFAError(-2, "split= needs sequences= or paged=: the fixed-length forward plans its own split.")
        if fp8 is not None and paged is None:
            raise MFAError(-2, "fp8= needs paged=: FP8 K/V is read from a paged cache only.")
        arr = (ctypes.c_void_p * MFA_BUFFER_COUNT)()
        for op, ptr in buffers.items():
            binding = AttentionOperand(op).bufferBinding
            if binding is None:
                raise MFAError(-2, f"Operand {AttentionOperand(op).name} has no buffer binding.")
            arr[binding] = ptr
        if fp8 is not None:
            _check(_lib.mfa_attention_kernel_encode_paged_fp8(self._handle, ctypes.byref(constants._c),
                                                              ctypes.byref(paged),
                                                              ctypes.byref(split) if split is not None else None,
                                                              ctypes.byref(fp8), ctypes.byref(arr),
                                                              ctypes.c_void_p(stream)))
        elif split is not None and paged is not None:
            _check(_lib.mfa_attention_kernel_encode_paged_split(self._handle, ctypes.byref(constants._c),
                                                                ctypes.byref(paged), ctypes.byref(split),
                                                                ctypes.byref(arr), ctypes.c_void_p(stream)))
        elif split is not None:
            _check(_lib.mfa_attention_kernel_encode_sequences_split(self._handle, ctypes.byref(constants._c),
                                                                    ctypes.byref(sequences), ctypes.byref(split),
                                                                    ctypes.byref(arr), ctypes.c_void_p(stream)))
        elif paged is not None:
            _check(_lib.mfa_attention_kernel_encode_paged(self._handle, ctypes.byref(constants._c), ctypes.byref(paged),
                                                          ctypes.byref(arr), ctypes.c_void_p(stream)))
        elif sequences is None:
            _check(_lib.mfa_attention_kernel_encode(self._handle, ctypes.byref(constants._c), ctypes.byref(arr),
                                                    ctypes.c_void_p(stream)))
        else:
            _check(_lib.mfa_attention_kernel_encode_sequences(self._handle, ctypes.byref(constants._c),
                                                              ctypes.byref(sequences), ctypes.byref(arr),
                                                              ctypes.c_void_p(stream)))


__all__ = [
    "AttentionDescriptor", "AttentionKernelDescriptor", "AttentionKernel", "AttentionKernelType",
    "AttentionOperand", "GEMMOperandPrecision", "FunctionConstantValues", "Backend", "MFAError", "SequenceTable", "PagedKV",
    "SplitKV", "SplitPlan", "FP8KV", "PagedKVAppend", "Rotary",
    "appendPagedKV", "library_path", "version", "setParameterTable", "hostAlloc", "hostFree", "bindThreadToDevice", "releaseDeviceResources",
]
