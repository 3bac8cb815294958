//
//  FlashAttention.swift -- drop-in Swift surface over the H100 C ABI.
//
//  Same public names, fields and failure behaviour as the reference package
//  (Sources/FlashAttention/Attention/*.swift), minus everything Metal-specific:
//    * `createSource()` is replaced by `encode(...)`: the kernels are ahead-of-time compiled CUDA, so
//      the compile + bind + dispatch the reference leaves to its caller happens behind the C ABI.
//    * `setFunctionConstants(_:)` fills a plain struct instead of MTLFunctionConstantValues.
//  Where the reference calls fatalError(...), so does this shim (with the C ABI's message).
//
import CMFAB200

/// GEMMOperandPrecision.swift:33-61 (raw values are shared with the C ABI).
public enum GEMMOperandPrecision: UInt16 {
  case FP32 = 0
  case FP16 = 1
  case BF16 = 2
  public var size: Int { self == .FP32 ? 4 : 2 }
  public var name: String { String(cString: mfa_precision_name(mfa_precision_t(UInt32(rawValue)))) }
}

/// AttentionKernelType.swift:8-23
public enum AttentionKernelType: UInt32 {
  case forward = 0
  case backwardQuery = 1
  case backwardKeyValue = 2
}

/// AttentionOperand.swift:8-72; raw values 0...9 are the buffer bindings.
public enum AttentionOperand: UInt32, Hashable, CustomStringConvertible {
  case Q = 0, K, V, O, L, D, dO, dV, dK, dQ, S, P, dP, dS
  public var description: String { String(cString: mfa_operand_name(mfa_operand_t(rawValue))) }
  public var bufferBinding: UInt8? {
    let binding = mfa_operand_buffer_binding(mfa_operand_t(rawValue))
    return binding < 0 ? nil : UInt8(binding)
  }
}

@inline(__always) private func check(_ status: Int32) {
  if status != 0 { fatalError(String(cString: mfa_last_error())) }
}

/// AttentionDescriptor.swift:10-27
public struct AttentionDescriptor {
  public var lowPrecisionInputs: Bool = false
  public var lowPrecisionIntermediates: Bool = false
  public var matrixDimensions: (row: UInt32, column: UInt32, head: UInt16)?
  public var transposeState: (Q: Bool, K: Bool, V: Bool, O: Bool)?
  /// library extension: BF16 Q/K/V/dO in memory (nil = the reference's FP16 policy).
  public var inputPrecisionOverride: GEMMOperandPrecision?
  /// library extension: number of independent single-head problems stored back to back.
  public var batchCount: UInt32 = 1
  /// library extension: causal mask aligned bottom-right (query row i sees key j iff j <= i + column - row); rows
  /// with no visible key get O = 0, L = +inf, D = 0, dQ = 0.
  public var causal: Bool = false

  public init() {}

  var c: mfa_attention_descriptor_t {
    var d = mfa_attention_descriptor_t()
    mfa_attention_descriptor_init(&d)
    d.low_precision_inputs = lowPrecisionInputs ? 1 : 0
    d.low_precision_intermediates = lowPrecisionIntermediates ? 1 : 0
    if let m = matrixDimensions {
      d.has_matrix_dimensions = 1
      d.row = m.row; d.column = m.column; d.head = m.head
    }
    if let t = transposeState {
      d.has_transpose_state = 1
      d.transpose_Q = t.Q ? 1 : 0; d.transpose_K = t.K ? 1 : 0
      d.transpose_V = t.V ? 1 : 0; d.transpose_O = t.O ? 1 : 0
    }
    d.input_precision_override = UInt8(inputPrecisionOverride?.rawValue ?? 0)
    d.batch_count = batchCount
    d.causal = causal ? 1 : 0
    return d
  }

  /// AttentionDescriptor.swift:33-130
  public func kernelDescriptor(type: AttentionKernelType) -> AttentionKernelDescriptor {
    var descriptor = c
    var output = AttentionKernelDescriptor()
    check(mfa_attention_descriptor_kernel_descriptor(&descriptor, mfa_kernel_type_t(type.rawValue), &output.c))
    return output
  }

  /// AttentionDescriptor+Precisions.swift:10-146
  public var memoryPrecisions: [AttentionOperand: GEMMOperandPrecision] {
    var descriptor = c
    var output: [AttentionOperand: GEMMOperandPrecision] = [:]
    for raw in UInt32(0)..<UInt32(MFA_BUFFER_COUNT) {
      var precision = mfa_precision_t(0)
      check(mfa_attention_descriptor_memory_precision(&descriptor, mfa_operand_t(raw), &precision))
      output[AttentionOperand(rawValue: raw)!] = GEMMOperandPrecision(rawValue: UInt16(precision.rawValue))!
    }
    return output
  }

  /// AttentionDescriptor+Precisions.swift:149-215.  P and dS read as the 16-bit input type whenever the tensor-core
  /// family serves the descriptor (they are MMA operands there) -- see `registerPrecisions` of the kernel descriptor
  /// for the per-kernel view.
  public var registerPrecisions: [AttentionOperand: GEMMOperandPrecision] {
    var descriptor = c
    var output: [AttentionOperand: GEMMOperandPrecision] = [:]
    for raw in UInt32(0)..<UInt32(MFA_OPERAND_COUNT) {
      var precision = mfa_precision_t(0)
      check(mfa_attention_descriptor_register_precision(&descriptor, mfa_operand_t(raw), &precision))
      output[AttentionOperand(rawValue: raw)!] = GEMMOperandPrecision(rawValue: UInt16(precision.rawValue))!
    }
    return output
  }

  /// AttentionDescriptor.swift:139-148 (R at index 0, C at index 1).  Writes kvGroup = 0 (no grouping).
  public func setFunctionConstants(_ constants: inout mfa_function_constants_t) {
    var descriptor = c
    check(mfa_attention_descriptor_set_function_constants(&descriptor, &constants))
  }

  /// The H100 parameter table this descriptor reads for `type` (AttentionDescriptor+Parameters.swift:106-285 format).
  public func parameterFile(type: AttentionKernelType) -> String {
    var descriptor = c
    return String(cString: mfa_attention_descriptor_parameter_file(&descriptor, mfa_kernel_type_t(type.rawValue)))
  }

  /// Elements of `operand`'s buffer (all `batchCount` problems).
  public func operandElements(_ operand: AttentionOperand) -> Int {
    var descriptor = c
    var count = 0
    check(mfa_attention_descriptor_operand_elements(&descriptor, mfa_operand_t(operand.rawValue), &count))
    return count
  }

  /// End-to-end call on HOST pointers (mfa_attention_run_host): H2D -> the selected kernels in the reference's order
  /// forward -> backwardQuery -> backwardKeyValue (SquareAttentionTest.swift:355-368) -> D2H, synchronous.
  public func runHost(types: [AttentionKernelType],
                      hostBuffers: [AttentionOperand: UnsafeMutableRawPointer],
                      device: Int32 = 0) {
    var descriptor = c
    var mask: UInt32 = 0
    for type in types { mask |= 1 << type.rawValue }
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in hostBuffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    check(mfa_attention_run_host(&descriptor, mask, &table, device))
  }
}

/// Page-locked host buffers on the GPU's NUMA node for `AttentionDescriptor.runHost` (library extension).
public enum HostMemory {
  /// `upload`: write-combined pages for buffers the host only writes and the GPU reads (Q, K, V, dO).
  public static func allocate(byteCount: Int, device: Int32 = 0, upload: Bool = false) -> UnsafeMutableRawPointer {
    var pointer: UnsafeMutableRawPointer?
    check(upload ? mfa_host_alloc_upload(byteCount, device, &pointer) : mfa_host_alloc(byteCount, device, &pointer))
    return pointer!
  }
  public static func free(_ pointer: UnsafeMutableRawPointer) { check(mfa_host_free(pointer)) }
  /// Pins the calling thread to the CPUs of the GPU's NUMA node; returns the node (-1: none reported).
  @discardableResult public static func bindThread(toDevice device: Int32) -> Int32 {
    var node: Int32 = -1
    check(mfa_host_bind_thread_to_device(device, &node))
    return node
  }
  /// Frees the library's scratch and workspaces on `device`.
  public static func releaseResources(device: Int32) { check(mfa_release_device_resources(device)) }
}

/// Which kernel family serves a descriptor (library extension; the reference has one family).
public enum AttentionBackend: UInt8 {
  case simtFP32 = 0
  case tcgen05 = 1
}

/// AttentionKernelDescriptor.swift:7-48 -- a plain, editable value.  Every field of the reference's struct is here,
/// readable and settable with the same types (optionals start as nil, dictionaries empty); storage is the C struct.
public struct AttentionKernelDescriptor {
  public var c = mfa_attention_kernel_descriptor_t()
  public init() { mfa_attention_kernel_descriptor_init(&c) }

  /// :8  blockDimensions
  public var blockDimensions: (parallelization: UInt16, traversal: UInt16, head: UInt16)? {
    get { c.has_block_dimensions == 0 ? nil : (c.block_parallelization, c.block_traversal, c.block_head) }
    set {
      c.has_block_dimensions = newValue == nil ? 0 : 1
      c.block_parallelization = newValue?.parallelization ?? 0
      c.block_traversal = newValue?.traversal ?? 0
      c.block_head = newValue?.head ?? 0
    }
  }

  /// :11  cacheState -- whether each operand stays resident on chip for the whole traversal
  public var cacheState: [AttentionOperand: Bool] {
    get {
      var output: [AttentionOperand: Bool] = [:]
      for raw in UInt32(0)..<UInt32(MFA_OPERAND_COUNT) where (c.cache_state_valid_mask >> UInt16(raw)) & 1 == 1 {
        output[AttentionOperand(rawValue: raw)!] = (c.cache_state_mask >> UInt16(raw)) & 1 == 1
      }
      return output
    }
    set {
      c.cache_state_valid_mask = 0
      c.cache_state_mask = 0
      for (operand, cached) in newValue {
        c.cache_state_valid_mask |= 1 << UInt16(operand.rawValue)
        if cached { c.cache_state_mask |= 1 << UInt16(operand.rawValue) }
      }
    }
  }

  /// :14  headDimension
  public var headDimension: UInt16? {
    get { c.has_head_dimension == 0 ? nil : c.head_dimension }
    set {
      c.has_head_dimension = newValue == nil ? 0 : 1
      c.head_dimension = newValue ?? 0
    }
  }

  private static func precisions(_ tuple: inout mfa_attention_kernel_descriptor_t,
                                 register: Bool) -> [AttentionOperand: GEMMOperandPrecision] {
    var output: [AttentionOperand: GEMMOperandPrecision] = [:]
    for raw in UInt32(0)..<UInt32(MFA_OPERAND_COUNT) {
      let value = mfa_attention_kernel_descriptor_get_precision(&tuple, mfa_operand_t(raw), register ? 1 : 0)
      if value >= 0 { output[AttentionOperand(rawValue: raw)!] = GEMMOperandPrecision(rawValue: UInt16(value))! }
    }
    return output
  }
  private static func setPrecisions(_ tuple: inout mfa_attention_kernel_descriptor_t, register: Bool,
                                    _ values: [AttentionOperand: GEMMOperandPrecision]) {
    for raw in UInt32(0)..<UInt32(MFA_OPERAND_COUNT) {
      let value = values[AttentionOperand(rawValue: raw)!].map { Int32($0.rawValue) } ?? -1
      mfa_attention_kernel_descriptor_set_precision(&tuple, mfa_operand_t(raw), register ? 1 : 0, value)
    }
  }

  /// :17  memoryPrecisions
  public var memoryPrecisions: [AttentionOperand: GEMMOperandPrecision] {
    get { var copy = c; return Self.precisions(&copy, register: false) }
    set { Self.setPrecisions(&c, register: false, newValue) }
  }
  /// :19  registerPrecisions
  public var registerPrecisions: [AttentionOperand: GEMMOperandPrecision] {
    get { var copy = c; return Self.precisions(&copy, register: true) }
    set { Self.setPrecisions(&c, register: true, newValue) }
  }

  /// :22  preferAsyncCache ("async" == TMA bulk-tensor copies on H100)
  public var preferAsyncCache: Bool? {
    get { c.prefer_async_cache == 0xFF ? nil : c.prefer_async_cache != 0 }
    set { c.prefer_async_cache = newValue.map { $0 ? 1 : 0 } ?? 0xFF }
  }
  /// :25  preferAsyncLoad
  public var preferAsyncLoad: Bool? {
    get { c.prefer_async_load == 0xFF ? nil : c.prefer_async_load != 0 }
    set { c.prefer_async_load = newValue.map { $0 ? 1 : 0 } ?? 0xFF }
  }

  /// :42  transposeState -- per operand; derivatives follow their forward operand (AttentionDescriptor.swift:96-111)
  public var transposeState: [AttentionOperand: Bool] {
    get {
      var output: [AttentionOperand: Bool] = [:]
      for raw in UInt32(0)..<UInt32(MFA_OPERAND_COUNT) where (c.transpose_state_valid_mask >> UInt16(raw)) & 1 == 1 {
        output[AttentionOperand(rawValue: raw)!] = (c.transpose_state_mask >> UInt16(raw)) & 1 == 1
      }
      return output
    }
    set {
      c.transpose_state_valid_mask = 0
      c.transpose_state_mask = 0
      for (operand, transposed) in newValue {
        c.transpose_state_valid_mask |= 1 << UInt16(operand.rawValue)
        if transposed { c.transpose_state_mask |= 1 << UInt16(operand.rawValue) }
      }
    }
  }

  /// :45  type
  public var type: AttentionKernelType? {
    get { c.type == 0xFF ? nil : AttentionKernelType(rawValue: UInt32(c.type)) }
    set { c.type = newValue.map { UInt8($0.rawValue) } ?? 0xFF }
  }

  /// library extension: the kernel family `AttentionDescriptor.kernelDescriptor(type:)` selected.
  public var backend: AttentionBackend {
    get { AttentionBackend(rawValue: c.backend) ?? .simtFP32 }
    set { c.backend = newValue.rawValue }
  }
  /// library extension: tuning columns of the parameter-table row, the small-grid split policy (minimum blocks per
  /// range, 0 = never; maximum ranges).
  public var splitPolicy: (minimumBlocks: UInt8, maximumSplits: UInt8) {
    get { (c.split_min_blocks, c.split_max) }
    set { c.split_min_blocks = newValue.minimumBlocks; c.split_max = newValue.maximumSplits }
  }

  /// library extension: the causal mask copied from AttentionDescriptor.causal (editable like the fields above).
  public var causal: Bool {
    get { c.causal != 0 }
    set { c.causal = newValue ? 1 : 0 }
  }
}

/// The parameter tables are data (AttentionDescriptor+Parameters.swift:106-285): replace the tensor-core family's table
/// of `type` at run time (`nil` restores the built-in one).
public func setParameterTable(type: AttentionKernelType, text: String?, transposed: Bool = false) {
  if let text = text {
    text.withCString { check(mfa_set_parameter_table(mfa_kernel_type_t(type.rawValue), transposed ? 1 : 0, $0)) }
  } else {
    check(mfa_set_parameter_table(mfa_kernel_type_t(type.rawValue), transposed ? 1 : 0, nil))
  }
}

/// AttentionKernel.swift:11-50, 268-363
public final class AttentionKernel {
  let handle: OpaquePointer
  let owned: Bool

  public init(descriptor: AttentionKernelDescriptor) {
    var kd = descriptor.c
    var out: OpaquePointer?
    check(mfa_attention_kernel_create(&kd, &out))
    handle = out!
    owned = true
  }
  /// Library-owned kernel object from the descriptor-keyed cache -- the analogue of
  /// `GEMMKernel.pipelineCache[descriptor]` (GEMMDescriptor+PipelineCache.swift:16-36).
  public init(cached descriptor: AttentionDescriptor, type: AttentionKernelType) {
    var d = descriptor.c
    var out: OpaquePointer?
    check(mfa_attention_kernel_cache_fetch(&d, mfa_kernel_type_t(type.rawValue), &out))
    handle = out!
    owned = false
  }
  /// A sliding window (left, right): with delta = column - row, query row i sees key j iff
  /// i + delta - left <= j <= i + delta + right, -1 leaving a side unbounded (mfa_attention_kernel_create_windowed).
  public init(descriptor: AttentionKernelDescriptor, window: (left: Int32, right: Int32)) {
    var kd = descriptor.c
    var w = mfa_attention_window_t(left: window.left, right: window.right)
    var out: OpaquePointer?
    check(mfa_attention_kernel_create_windowed(&kd, &w, &out))
    handle = out!
    owned = true
  }
  /// The cached kernel object of (descriptor, type, window) (mfa_attention_kernel_cache_fetch_windowed).
  public init(cached descriptor: AttentionDescriptor, type: AttentionKernelType, window: (left: Int32, right: Int32)) {
    var d = descriptor.c
    var w = mfa_attention_window_t(left: window.left, right: window.right)
    var out: OpaquePointer?
    check(mfa_attention_kernel_cache_fetch_windowed(&d, mfa_kernel_type_t(type.rawValue), &w, &out))
    handle = out!
    owned = false
  }
  deinit { if owned { mfa_attention_kernel_destroy(handle) } }

  public var blockDimensions: (parallelization: UInt16, traversal: UInt16, head: UInt16) {
    var out: (UInt16, UInt16, UInt16) = (0, 0, 0)
    withUnsafeMutablePointer(to: &out) {
      $0.withMemoryRebound(to: UInt16.self, capacity: 3) { check(mfa_attention_kernel_block_dimensions(handle, $0)) }
    }
    return out
  }
  public var threadgroupSize: UInt32 {
    var out: UInt32 = 0
    check(mfa_attention_kernel_threadgroup_size(handle, &out))
    return out
  }
  public var threadgroupMemoryAllocation: UInt32 {
    var out: UInt32 = 0
    check(mfa_attention_kernel_threadgroup_memory_allocation(handle, &out))
    return out
  }

  /// Thread blocks along the parallelization dimension (R for forward / backwardQuery, C for backwardKeyValue) times
  /// the batch: what the reference's caller computes for dispatchThreadgroups (SquareAttentionTest.swift:328-339).
  public func gridSize(constants: mfa_function_constants_t) -> UInt32 {
    var constants = constants
    var out: UInt32 = 0
    check(mfa_attention_kernel_grid_size(handle, &constants, &out))
    return out
  }
  /// CUDA kernels one `encode` launches (2 only when a small grid is split and a merge kernel follows).
  public func launchCount(constants: mfa_function_constants_t) -> UInt32 {
    var constants = constants
    var out: UInt32 = 0
    check(mfa_attention_kernel_launch_count(handle, &constants, &out))
    return out
  }
  /// Stands in for `createSource()` (AttentionKernel+Source.swift:11-55): the name of the ahead-of-time compiled kernel.
  public var sourceName: String { String(cString: mfa_attention_kernel_source_name(handle)) }

  /// What the reference's callers do by hand around `createSource()` (SquareAttentionTest.swift:240-372):
  /// `buffers[binding]` are DEVICE pointers at AttentionOperand.bufferBinding; `stream` is a cudaStream_t.
  public func encode(constants: mfa_function_constants_t,
                     buffers: [AttentionOperand: UnsafeMutableRawPointer],
                     stream: UnsafeMutableRawPointer? = nil) {
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in buffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    var constants = constants
    check(mfa_attention_kernel_encode(handle, &constants, &table, stream))
  }

  // ---- library extension: packed variable-length sequences (mfa_sequence_table_t, FlashAttention's cu_seqlens)
  public func gridSize(constants: mfa_function_constants_t, sequences: SequenceTable) -> UInt32 {
    var constants = constants
    var sequences = sequences
    var out: UInt32 = 0
    check(mfa_attention_kernel_grid_size_sequences(handle, &constants, &sequences, &out))
    return out
  }
  public func launchCount(constants: mfa_function_constants_t, sequences: SequenceTable) -> UInt32 {
    var constants = constants
    var sequences = sequences
    var out: UInt32 = 0
    check(mfa_attention_kernel_launch_count_sequences(handle, &constants, &sequences, &out))
    return out
  }
  /// `encode` over the sequences of `sequences`: every problem's rows are cut into the sequences of the device offset
  /// tables, and each sequence attends only to its own keys.
  public func encode(constants: mfa_function_constants_t, sequences: SequenceTable,
                     buffers: [AttentionOperand: UnsafeMutableRawPointer],
                     stream: UnsafeMutableRawPointer? = nil) {
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in buffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    var constants = constants
    var sequences = sequences
    check(mfa_attention_kernel_encode_sequences(handle, &constants, &sequences, &table, stream))
  }

  // ---- library extension: the forward over a paged K/V cache (mfa_paged_kv_t, vLLM's block table)
  public func gridSize(constants: mfa_function_constants_t, paged: PagedKV) -> UInt32 {
    var constants = constants
    var paged = paged
    var out: UInt32 = 0
    check(mfa_attention_kernel_grid_size_paged(handle, &constants, &paged, &out))
    return out
  }
  public func launchCount(constants: mfa_function_constants_t, paged: PagedKV) -> UInt32 {
    var constants = constants
    var paged = paged
    var out: UInt32 = 0
    check(mfa_attention_kernel_launch_count_paged(handle, &constants, &paged, &out))
    return out
  }
  /// The forward `encode` over a paged K/V cache: the K and V buffers are page pools [pages][pageSize][Hkv][D], read in
  /// place through the device page table.
  public func encode(constants: mfa_function_constants_t, paged: PagedKV,
                     buffers: [AttentionOperand: UnsafeMutableRawPointer],
                     stream: UnsafeMutableRawPointer? = nil) {
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in buffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    var constants = constants
    var paged = paged
    check(mfa_attention_kernel_encode_paged(handle, &constants, &paged, &table, stream))
  }

  // ---- library extension: the split-KV forward over packed sequences or a paged cache (mfa_split_kv_t)
  public func splitPlan(constants: mfa_function_constants_t, sequences: SequenceTable, split: SplitKV) -> SplitPlan {
    var constants = constants
    var sequences = sequences
    var split = split
    var out = SplitPlan()
    check(mfa_attention_kernel_split_plan(handle, &constants, &sequences, nil, &split, &out))
    return out
  }
  public func splitPlan(constants: mfa_function_constants_t, paged: PagedKV, split: SplitKV) -> SplitPlan {
    var constants = constants
    var paged = paged
    var split = split
    var out = SplitPlan()
    check(mfa_attention_kernel_split_plan(handle, &constants, nil, &paged, &split, &out))
    return out
  }
  /// The forward `encode` over `sequences` whose key range may be split across CTAs (`split`).
  public func encode(constants: mfa_function_constants_t, sequences: SequenceTable, split: SplitKV,
                     buffers: [AttentionOperand: UnsafeMutableRawPointer],
                     stream: UnsafeMutableRawPointer? = nil) {
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in buffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    var constants = constants
    var sequences = sequences
    var split = split
    check(mfa_attention_kernel_encode_sequences_split(handle, &constants, &sequences, &split, &table, stream))
  }
  /// The forward `encode` over a paged K/V cache whose key range may be split across CTAs (`split`).
  public func encode(constants: mfa_function_constants_t, paged: PagedKV, split: SplitKV,
                     buffers: [AttentionOperand: UnsafeMutableRawPointer],
                     stream: UnsafeMutableRawPointer? = nil) {
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in buffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    var constants = constants
    var paged = paged
    var split = split
    check(mfa_attention_kernel_encode_paged_split(handle, &constants, &paged, &split, &table, stream))
  }
  /// The forward `encode` over a paged cache whose K and V pools hold FP8 E4M3 bytes with per-K/V-head scales
  /// (`fp8`); `split` nil runs it unsplit, as `encode(constants:paged:buffers:)`.
  public func encode(constants: mfa_function_constants_t, paged: PagedKV, split: SplitKV?, fp8: FP8KV,
                     buffers: [AttentionOperand: UnsafeMutableRawPointer],
                     stream: UnsafeMutableRawPointer? = nil) {
    var table = [UnsafeMutableRawPointer?](repeating: nil, count: Int(MFA_BUFFER_COUNT))
    for (operand, pointer) in buffers {
      guard let binding = operand.bufferBinding else { fatalError("Operand \(operand) has no buffer binding.") }
      table[Int(binding)] = pointer
    }
    var constants = constants
    var paged = paged
    var fp8 = fp8
    if var split = split {
      check(mfa_attention_kernel_encode_paged_fp8(handle, &constants, &paged, &split, &fp8, &table, stream))
    } else {
      check(mfa_attention_kernel_encode_paged_fp8(handle, &constants, &paged, nil, &fp8, &table, stream))
    }
  }
}

/// library extension: a split-KV forward.  `numSplits` 0 lets the library plan, 1...16 is taken as given;
/// `maxColumn` is a planning hint bounding every sequence's keys (0 = the table's bound).
public typealias SplitKV = mfa_split_kv_t
extension mfa_split_kv_t {
  public init(numSplits: UInt32 = 0, maxColumn: UInt32 = 0) {
    self.init(num_splits: numSplits, max_column: maxColumn)
  }
}
/// library extension: what a split-KV encode launches (splits, heads_per_tile, grid_size, launch_count).
public typealias SplitPlan = mfa_split_plan_t

/// library extension: packed variable-length sequences.  `rowOffsets` / `columnOffsets` are DEVICE pointers to
/// `count + 1` Int32 entries each; `maxRow` / `maxColumn` are at least every sequence's query / key length.
public typealias SequenceTable = mfa_sequence_table_t
extension mfa_sequence_table_t {
  public init(count: UInt32, maxRow: UInt32, maxColumn: UInt32, rowOffsets: UnsafePointer<Int32>,
              columnOffsets: UnsafePointer<Int32>) {
    self.init(count: count, max_row: maxRow, max_column: maxColumn, row_offsets: rowOffsets,
              column_offsets: columnOffsets)
  }
}

/// library extension: a paged K/V cache.  `rowOffsets` (count + 1), `columnLengths` (count) and `pageTable`
/// (count x pageStride) are DEVICE pointers to Int32 entries; `maxRow` is at least every sequence's query count and
/// `pageSize` a power of two >= 16.
public typealias PagedKV = mfa_paged_kv_t
extension mfa_paged_kv_t {
  public init(count: UInt32, maxRow: UInt32, rowOffsets: UnsafePointer<Int32>, columnLengths: UnsafePointer<Int32>,
              pageTable: UnsafePointer<Int32>, pageStride: UInt32, pageSize: UInt32) {
    self.init(count: count, max_row: maxRow, row_offsets: rowOffsets, column_lengths: columnLengths,
              page_table: pageTable, page_stride: pageStride, page_size: pageSize)
  }
}

/// library extension: grouped-query / multi-query attention, a launch-time constant like R, C and the batch.  The
/// query problems per K/V problem (0 or 1: none shared); query problem b reads K/V problem b / kvGroup, and dK / dV
/// are summed per group.  `setFunctionConstants` writes 0: set it afterwards (Hq / Hkv).
extension mfa_function_constants_t {
  public var kvGroup: UInt32 {
    get { kv_group }
    set { kv_group = newValue }
  }
}

/// library extension: FP8 E4M3 K/V pools of a paged forward, with one FP32 scale per K/V head in device memory
/// (`kScale`, `vScale`: batch_count / kv_group entries each; nil means every scale is 1).
public typealias FP8KV = mfa_fp8_kv_t
extension mfa_fp8_kv_t {
  public init(kScale: UnsafePointer<Float>? = nil, vScale: UnsafePointer<Float>? = nil) {
    self.init(k_scale: kScale, v_scale: vScale)
  }
}

/// library extension: the new tokens of a paged K/V append.  `kNew` / `vNew` are DEVICE pointers, token t's K/V head
/// kv at element t * tokenStride + kv * headDimension (tokenStride 0: kvHeads * headDimension); `rows` is the tokens
/// they hold, `poolRows` the rows of each pool (num_pages * page_size), `precision` the element type of kNew / vNew.
public typealias PagedKVAppend = mfa_paged_kv_append_t
extension mfa_paged_kv_append_t {
  public init(kNew: UnsafeRawPointer, vNew: UnsafeRawPointer, rows: UInt32, tokenStride: UInt32 = 0, kvHeads: UInt32,
              headDimension: UInt32, poolRows: UInt32, precision: GEMMOperandPrecision) {
    self.init(k_new: kNew, v_new: vNew, rows: rows, token_stride: tokenStride, kv_heads: kvHeads,
              head_dimension: headDimension, pool_rows: poolRows, precision: UInt32(precision.rawValue))
  }
}

/// library extension: writes a step's new keys and values into the page pools through the table of the step's paged
/// forward (new token i of sequence s becomes key columnLengths[s] - Rs + i).  `fp8` nil: the pools hold
/// `append.precision` elements, copied bit for bit; otherwise E4M3 bytes, each value divided by its K/V head's scale and
/// saturated to +-448.  One launch on `stream`, capturable into a CUDA graph with the forward.
public func appendPagedKV(paged: PagedKV, append: PagedKVAppend, kPool: UnsafeMutableRawPointer,
                          vPool: UnsafeMutableRawPointer, fp8: FP8KV? = nil, stream: UnsafeMutableRawPointer? = nil) {
  var paged = paged
  var append = append
  if var fp8 = fp8 {
    check(mfa_paged_kv_append(&paged, &append, kPool, vPool, &fp8, stream))
  } else {
    check(mfa_paged_kv_append(&paged, &append, kPool, vPool, nil, stream))
  }
}

/// library extension: rotary position embedding for a paged K/V append.  `qNew` is a DEVICE pointer, token t's query
/// head h at element t * qTokenStride + h * headDimension (qTokenStride 0: queryHeads * headDimension), in the append's
/// precision; `qOut` the paged forward's Q buffer [queryHeads][rows][headDimension]; `cos` / `sin` Float tables in device
/// memory, position p, frequency j < rotaryDim / 2 at p * tableStride + j (tableStride 0: rotaryDim / 2), `positions`
/// rows of them (at least pageStride * pageSize); `interleaved` pairs (2j, 2j + 1) (GPT-J), else (j, j + rotaryDim / 2).
public typealias Rotary = mfa_rotary_t
extension mfa_rotary_t {
  public init(qNew: UnsafeRawPointer, qOut: UnsafeMutableRawPointer, cos: UnsafePointer<Float>,
              sin: UnsafePointer<Float>, queryHeads: UInt32, qTokenStride: UInt32 = 0, rotaryDim: UInt32,
              tableStride: UInt32 = 0, positions: UInt32, interleaved: Bool = false) {
    self.init(q_new: qNew, q_out: qOut, cos: cos, sin: sin, query_heads: queryHeads, q_token_stride: qTokenStride,
              rotary_dim: rotaryDim, table_stride: tableStride, positions: positions, interleaved: interleaved ? 1 : 0)
  }
}

/// library extension: `appendPagedKV` with the queries and new keys rotated by RoPE at their cache positions, and the
/// queries written to `rotary.qOut` in the paged forward's layout, in the same launch.
public func appendPagedKV(paged: PagedKV, append: PagedKVAppend, rotary: Rotary, kPool: UnsafeMutableRawPointer,
                          vPool: UnsafeMutableRawPointer, fp8: FP8KV? = nil, stream: UnsafeMutableRawPointer? = nil) {
  var paged = paged
  var append = append
  var rotary = rotary
  if var fp8 = fp8 {
    check(mfa_paged_kv_append_rotary(&paged, &append, &rotary, kPool, vPool, &fp8, stream))
  } else {
    check(mfa_paged_kv_append_rotary(&paged, &append, &rotary, kPool, vPool, nil, stream))
  }
}
