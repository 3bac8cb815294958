"""Host-side logic of the C ABI (no GPU): descriptor -> kernel-descriptor heuristic, precision policy,
parameter tables, validation / error behaviour, and that libmfa_b200.so exports every symbol the header
declares.  Mirrors what the reference's Swift types do on the CPU
(Sources/FlashAttention/Attention/AttentionDescriptor/*.swift, AttentionKernel.swift)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

import mfa_b200 as mfa
from mfa_b200 import AttentionKernelType as KT
from mfa_b200 import AttentionOperand as Op
from mfa_b200 import GEMMOperandPrecision as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make(row=64, column=64, head=32, lowIn=False, lowMid=False, transposes=(False,) * 4, bf16=False):
    d = mfa.AttentionDescriptor()
    d.lowPrecisionInputs, d.lowPrecisionIntermediates = lowIn, lowMid
    d.matrixDimensions = (row, column, head)
    d.transposeState = transposes
    if bf16:
        d.inputPrecisionOverride = P.BF16
    return d


def test_header_symbols_are_exported():
    header = open(os.path.join(ROOT, "include", "mfa_b200.h")).read()
    declared = set(re.findall(r"MFA_API\s+[\w\s\*]+?\b(mfa_\w+)\s*\(", header))
    assert len(declared) >= 20
    nm = subprocess.check_output(["nm", "-D", "--defined-only", mfa.library_path()], text=True)
    exported = set(re.findall(r"\b(mfa_\w+)\b", nm))
    missing = declared - exported
    assert not missing, f"declared in include/mfa_b200.h but not exported: {sorted(missing)}"
    lib = ctypes.CDLL(mfa.library_path())
    for name in declared:
        assert getattr(lib, name) is not None


def test_enum_raw_values_match_reference():
    assert (P.FP32, P.FP16, P.BF16) == (0, 1, 2)                     # GEMMOperandPrecision.swift:33-37
    assert [P.FP32.size, P.FP16.size, P.BF16.size] == [4, 2, 2]      # :51-60
    bindings = {Op.Q: 0, Op.K: 1, Op.V: 2, Op.O: 3, Op.L: 4, Op.D: 5, Op.dO: 6, Op.dV: 7, Op.dK: 8, Op.dQ: 9}
    for op, slot in bindings.items():                                 # AttentionOperand.swift:52-71
        assert op.bufferBinding == slot
    for op in (Op.S, Op.P, Op.dP, Op.dS):
        assert op.bufferBinding is None


def test_memory_precisions_follow_reference_policy():
    """AttentionDescriptor+Precisions.swift:10-146."""
    m = make().memoryPrecisions
    assert all(m[op] == P.FP32 for op in m)
    m = make(lowIn=True).memoryPrecisions
    assert (m[Op.Q], m[Op.K], m[Op.V], m[Op.dO]) == (P.FP16, P.FP16, P.FP16, P.BF16)
    assert (m[Op.L], m[Op.D]) == (P.FP32, P.FP32)
    m = make(lowMid=True).memoryPrecisions
    assert (m[Op.Q], m[Op.L], m[Op.D]) == (P.FP32, P.FP16, P.BF16)
    for flags in ((True, True), (True, False), (False, True)):
        m = make(lowIn=flags[0], lowMid=flags[1]).memoryPrecisions
        assert all(m[op] == P.FP32 for op in (Op.O, Op.dV, Op.dK, Op.dQ))   # :140-143 outputs always FP32
    m = make(lowIn=True, bf16=True).memoryPrecisions                         # library extension
    assert (m[Op.Q], m[Op.K], m[Op.V], m[Op.dO]) == (P.BF16,) * 4


def test_register_precisions():
    # a descriptor the FP32 CUDA-core family serves (head beyond the tensor-core kernels): the reference's policy verbatim
    assert make(head=300, lowIn=True).kernelDescriptor(KT.forward).backend == mfa.Backend.simtFP32
    r = make(head=300, lowIn=True, lowMid=True).registerPrecisions
    assert r[Op.O] == r[Op.dV] == r[Op.dK] == r[Op.dQ] == P.FP32            # :209-212
    assert r[Op.dS] == P.BF16 and r[Op.dP] == P.FP32 and r[Op.P] == P.FP16  # :198-200 (native BF16 branch)
    r = make(head=300, lowIn=True, lowMid=False).registerPrecisions
    assert r[Op.P] == P.FP32 and r[Op.dS] == P.FP32                         # :203-205
    r = make().registerPrecisions
    assert all(v == P.FP32 for v in r.values())


def test_register_precisions_report_what_the_tensor_core_kernels_do():
    """On the tensor-core family P and dS are MMA operands: always the 16-bit input element type, whatever
    lowPrecisionIntermediates says (documented deviation from AttentionDescriptor+Precisions.swift:203-205) -- the
    descriptor must not advertise FP32 registers the kernel does not have."""
    for lowMid in (False, True):
        d = make(head=64, lowIn=True, lowMid=lowMid)
        assert d.kernelDescriptor(KT.forward).backend == mfa.Backend.tcgen05
        r = d.registerPrecisions
        assert r[Op.P] == P.FP16 and r[Op.dS] == P.FP16 and r[Op.dP] == P.FP32 and r[Op.S] == P.FP32
        for t in KT:
            kd = d.kernelDescriptor(t).registerPrecisions
            assert kd[Op.P] == P.FP16 and kd[Op.dS] == P.FP16
        rb = make(head=64, lowIn=True, lowMid=lowMid, bf16=True).registerPrecisions
        assert rb[Op.P] == P.BF16 and rb[Op.dS] == P.BF16


def test_incomplete_descriptor_is_an_error_not_a_crash():
    d = mfa.AttentionDescriptor()
    with pytest.raises(mfa.MFAError, match="Descriptor was incomplete"):     # AttentionDescriptor.swift:89-91
        d.kernelDescriptor(KT.forward)
    d.matrixDimensions = (8, 8, 8)
    with pytest.raises(mfa.MFAError, match="Descriptor was incomplete"):     # transposeState still nil (:96-99)
        d.kernelDescriptor(KT.forward)
    with pytest.raises(mfa.MFAError, match="Descriptor was incomplete"):     # AttentionKernel.swift:28-34
        mfa.AttentionKernel(mfa.AttentionKernelDescriptor())


def test_kernel_descriptor_fields():
    d = make(row=300, column=200, head=77, transposes=(True, False, True, False))
    for t in KT:
        kd = d.kernelDescriptor(t)
        par, trav, head = kd.blockDimensions
        assert head <= (77 + 7) // 8 * 8                                      # AttentionDescriptor.swift:41-54
        assert kd.headDimension == 77 and kd.type == t
        ts = kd.transposeState                                               # :96-111 derivatives mirror inputs
        assert ts[Op.Q] and ts[Op.dQ] and ts[Op.V] and ts[Op.dV]
        assert not ts[Op.K] and not ts[Op.dK] and not ts[Op.O] and not ts[Op.dO]
        assert kd.backend == mfa.Backend.simtFP32
    expected = {KT.forward: {Op.Q, Op.O}, KT.backwardQuery: {Op.Q, Op.dO, Op.dQ},
                KT.backwardKeyValue: {Op.K, Op.V, Op.dV, Op.dK}}                # :58-66
    for t, ops in expected.items():
        assert set(d.kernelDescriptor(t).cacheState) == ops


def test_heuristic_selects_tensor_core_family_only_where_it_applies():
    assert make(4096, 4096, 128, lowIn=True, bf16=True).kernelDescriptor(KT.forward).backend == mfa.Backend.tcgen05
    assert make(4096, 4096, 64, lowIn=True).kernelDescriptor(KT.forward).backend == mfa.Backend.tcgen05
    assert make(4096, 4096, 128).kernelDescriptor(KT.forward).backend == mfa.Backend.simtFP32       # FP32 inputs
    # D % 8 != 0 with 16-bit row-major operands: tensor cores through head-dimension padding (kernels/pad_head.cu) ...
    kd77 = make(64, 64, 77, lowIn=True).kernelDescriptor(KT.forward)
    assert kd77.backend == mfa.Backend.tcgen05 and kd77.headDimension == 77 and kd77.blockDimensions[2] == 80
    assert make(64, 64, 77, lowIn=True).kernelDescriptor(KT.backwardKeyValue).backend == mfa.Backend.tcgen05
    # ... as far as the kernels reach (pad8(D) <= 256), and not for transposed operands
    assert make(64, 64, 199, lowIn=True).kernelDescriptor(KT.forward).backend == mfa.Backend.tcgen05
    kd199 = make(64, 64, 199, lowIn=True).kernelDescriptor(KT.backwardQuery)
    assert kd199.backend == mfa.Backend.tcgen05 and kd199.blockDimensions == (64, 64, 200)   # wide-head dQ: one warpgroup
    assert make(64, 64, 260, lowIn=True).kernelDescriptor(KT.backwardQuery).backend == mfa.Backend.simtFP32
    assert make(64, 64, 260, lowIn=True).kernelDescriptor(KT.forward).backend == mfa.Backend.simtFP32
    assert make(64, 64, 77, lowIn=True, transposes=(True, False, False, False)).kernelDescriptor(
        KT.forward).backend == mfa.Backend.simtFP32
    # transposed operands: staged row-major for the tensor-core kernels where the transposed view has a 16-byte row pitch
    # (sequence length a multiple of 8 elements)
    tK = make(64, 64, 64, lowIn=True, transposes=(False, True, False, False))
    assert tK.kernelDescriptor(KT.forward).backend == mfa.Backend.tcgen05
    assert tK.kernelDescriptor(KT.forward).blockDimensions == (128, 128, 64)
    for t in (KT.backwardQuery, KT.backwardKeyValue):
        assert tK.kernelDescriptor(t).backend == mfa.Backend.tcgen05
        assert tK.kernelDescriptor(t).blockDimensions == (128, 64, 64)       # 64-row traversal blocks
        mfa.AttentionKernel(tK.kernelDescriptor(t))                           # ... and the kernel object accepts them
    # backward: Q^T and dO^T (which follows O) are addressed through R, K^T and V^T through C
    assert make(77, 64, 64, lowIn=True, transposes=(False, False, False, True)).kernelDescriptor(
        KT.backwardKeyValue).backend == mfa.Backend.simtFP32
    assert make(64, 77, 64, lowIn=True, transposes=(False, False, False, True)).kernelDescriptor(
        KT.backwardKeyValue).backend == mfa.Backend.tcgen05
    assert make(64, 77, 64, lowIn=True, transposes=(False, True, False, False)).kernelDescriptor(
        KT.forward).backend == mfa.Backend.simtFP32                                                # C % 8 != 0
    assert make(77, 64, 64, lowIn=True, transposes=(False, True, False, True)).kernelDescriptor(
        KT.forward).backend == mfa.Backend.tcgen05                                                 # only K's pitch matters
    assert make(77, 64, 64, lowIn=True, transposes=(True, False, False, False)).kernelDescriptor(
        KT.forward).backend == mfa.Backend.simtFP32                                                # R % 8 != 0
    # the kernel cache must not hand the tcgen05 kernel of an aligned shape to an unaligned one
    a = mfa.AttentionKernel.cached(make(64, 64, 64, lowIn=True, transposes=(True, False, False, False)), KT.forward)
    b = mfa.AttentionKernel.cached(make(77, 64, 64, lowIn=True, transposes=(True, False, False, False)), KT.forward)
    assert a._handle.value != b._handle.value and "tcgen05" in a.sourceName() and "simt" in b.sourceName()
    kd = make(4096, 4096, 128, lowIn=True, bf16=True).kernelDescriptor(KT.forward)
    assert kd.preferAsyncLoad and kd.preferAsyncCache           # "async" == TMA on H100
    assert kd.cacheState == {Op.Q: True, Op.O: True}             # Q resident in SMEM, O resident in registers


def test_parameter_file_has_reference_format():
    text = make(4096, 4096, 128, lowIn=True, bf16=True).parameterFile(KT.forward)
    rows = [line for line in text.split("\n") if line.strip()]
    # the reference's five segments (AttentionParameterRow.swift:46-49) + three tuning columns on the tensor-core family
    assert rows and all(len([c for c in row.split("|") if c != ""]) == 8 for row in rows)
    simt = make(64, 64, 35).parameterFile(KT.forward)
    assert all(len([c for c in row.split("|") if c != ""]) == 5 for row in simt.split("\n") if row.strip())
    maxima = [int(row.split("|")[1]) for row in rows]
    assert maxima == sorted(maxima)


def test_kernel_object_reports_launch_geometry():
    d = make(4096, 4096, 128, lowIn=True, bf16=True)
    d.batchCount = 64
    k = mfa.AttentionKernel(d.kernelDescriptor(KT.forward))
    c = mfa.FunctionConstantValues()
    d.setFunctionConstants(c)
    assert (c.row, c.column, c.batchCount) == (4096, 4096, 64)              # AttentionDescriptor.swift:144-147
    par, trav, head = k.blockDimensions
    assert k.gridSize(c) == (4096 + par - 1) // par * 64                      # SquareAttentionTest.swift:328-339
    assert k.threadgroupSize % 32 == 0 and 0 < k.threadgroupMemoryAllocation <= 232448
    assert "tcgen05" in k.sourceName() and k.launchCount(c) >= 1
    k2 = mfa.AttentionKernel(make(10, 10, 3).kernelDescriptor(KT.backwardKeyValue))
    assert "simt" in k2.sourceName()


def test_invalid_precision_pairs_are_rejected():
    kd = make(lowIn=True).kernelDescriptor(KT.forward)
    kd.setRegisterPrecision(Op.Q, P.BF16)                                      # FP16 memory -> BF16 register
    with pytest.raises(mfa.MFAError, match="Invalid precisions"):             # AttentionKernel.swift:90-105
        mfa.AttentionKernel(kd)
    kd = make().kernelDescriptor(KT.forward)
    kd.setMemoryPrecision(Op.K, None)
    with pytest.raises(mfa.MFAError, match="was not specified"):
        mfa.AttentionKernel(kd)


def test_edited_descriptor_outside_compiled_kernels_is_rejected():
    kd = make(lowIn=True, head=64).kernelDescriptor(KT.forward)
    kd.blockDimensions = (32, 80, 16)                                          # an Apple tile shape
    with pytest.raises(mfa.MFAError, match="no compiled sm_90a kernel"):
        mfa.AttentionKernel(kd)
    with pytest.raises(mfa.MFAError, match="exceeds 512"):
        mfa.AttentionKernel(make(head=600).kernelDescriptor(KT.forward))


def test_encode_without_gpu_fails_loudly_instead_of_falling_back():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    d = make(8, 8, 8)
    k = mfa.AttentionKernel(d.kernelDescriptor(KT.forward))
    c = mfa.FunctionConstantValues()
    d.setFunctionConstants(c)
    with pytest.raises(mfa.MFAError) as err:
        k.encode(c, {Op.Q: 16, Op.K: 16, Op.V: 16, Op.O: 16, Op.L: 16})
    assert err.value.status == -6 and "no CPU fallback" in str(err.value)      # MFA_ERROR_NO_DEVICE
    with pytest.raises(mfa.MFAError):
        d.runHost([KT.forward], {}, device=0)


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under the product package may import, link or call it."""
    pkg = os.path.join(ROOT, "metal-flash-attention_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".h", ".hpp", ".swift")) or f == "Makefile":
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in text.lower().replace("test infrastructure", ""), os.path.join(dirpath, f)
    ldd = subprocess.check_output(["ldd", mfa.library_path()], text=True)
    assert "oracle" not in ldd


def test_kernel_cache_returns_one_object_per_descriptor_and_type():
    """mfa_attention_kernel_cache_fetch (the analogue of GEMMKernel.pipelineCache, GEMMDescriptor+PipelineCache.swift:
    16-36): R, C and the batch count are launch constants, not part of the key; head, precisions, transposes are."""
    before = mfa.AttentionKernel.cacheSize()
    a = mfa.AttentionKernel.cached(make(4096, 4096, 120, lowIn=True, bf16=True), KT.forward)
    b = mfa.AttentionKernel.cached(make(512, 77, 120, lowIn=True, bf16=True), KT.forward)       # other R, C: same kernel
    assert a._handle.value == b._handle.value and mfa.AttentionKernel.cacheSize() == before + 1
    c = mfa.AttentionKernel.cached(make(4096, 4096, 120, lowIn=True, bf16=True), KT.backwardQuery)
    d = mfa.AttentionKernel.cached(make(4096, 4096, 120, lowIn=True), KT.forward)                 # FP16 inputs
    e = mfa.AttentionKernel.cached(make(4096, 4096, 112, lowIn=True, bf16=True), KT.forward)      # other head dimension
    assert len({a._handle.value, c._handle.value, d._handle.value, e._handle.value}) == 4
    assert mfa.AttentionKernel.cacheSize() == before + 4
    assert a.blockDimensions == mfa.AttentionKernel(make(4096, 4096, 120, lowIn=True, bf16=True).kernelDescriptor(
        KT.forward)).blockDimensions
    del a, b, c, d, e                                  # library-owned handles: dropping the wrappers must not free them
    again = mfa.AttentionKernel.cached(make(4096, 4096, 120, lowIn=True, bf16=True), KT.forward)
    assert again.threadgroupSize == 256 and mfa.AttentionKernel.cacheSize() == before + 4
    with pytest.raises(mfa.MFAError, match="Descriptor was incomplete"):
        mfa.AttentionKernel.cached(mfa.AttentionDescriptor(), KT.forward)


def test_reference_low_precision_policy_maps_to_the_tensor_core_family():
    """FP16 Q/K/V + BF16 dO (AttentionDescriptor+Precisions.swift:13-23) is served by the tcgen05 kernels for all three
    kernel types (the backward kernels convert the staged dO tiles on chip)."""
    for lowMid in (False, True):
        d = make(2048, 2048, 64, lowIn=True)
        d.lowPrecisionIntermediates = lowMid
        assert d.memoryPrecisions[Op.dO] == mfa.GEMMOperandPrecision.BF16
        for t in KT:
            kd = d.kernelDescriptor(t)
            assert kd.backend == mfa.Backend.tcgen05
            assert "tcgen05" in mfa.AttentionKernel(kd).sourceName()


def test_cpp_host_mirror_compiles_and_links_against_the_c_abi(tmp_path):
    """metal-flash-attention_b200/host/FlashAttention.hpp (the compiled-language host layer standing in for the
    reference's Swift package) builds with g++ against include/mfa_b200.h + libmfa_b200.so and reproduces the
    descriptor -> kernel flow, including the reference's fatalError message for an incomplete descriptor."""
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  AttentionDescriptor d;
  d.lowPrecisionInputs = true;
  d.matrixDimensions = MatrixDimensions{4096, 4096, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  AttentionKernel k(d.kernelDescriptor(AttentionKernelType::forward));
  auto [par, trav, head] = k.blockDimensions();
  AttentionKernel cached(d, AttentionKernelType::backwardKeyValue);
  std::printf("%u %u %u %u %u\n", par, trav, head, k.threadgroupSize(), cached.threadgroupSize());
  try {
    AttentionDescriptor incomplete;
    incomplete.kernelDescriptor(AttentionKernelType::forward);
  } catch (const std::runtime_error &e) {
    std::printf("%s\n", e.what());
  }
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).splitlines()
    assert out[0] == "128 128 128 256 256" and out[1] == "Descriptor was incomplete."


FORWARD_TABLE = ("| 64  | 128 | 128 | 64  | Q, O | 2 | 8 | 4 |\n"
                 "| 128 | 128 | 128 | 128 | Q, O | 1 | 2 | 16 |\n"
                 "| 256 | 128 | 64  | 256 | Q, O | 0 | 0 | 1 |\n")


def test_parameter_table_is_live_data():
    """The H100 parameter table drives the kernel (AttentionDescriptor+Parameters.swift:106-285 analogue): editing a row
    changes the kernel descriptor, the cached kernel object and the small-grid split policy; every compiled variant is
    accepted, anything else is rejected and leaves the current table in place."""
    d = make(4096, 4096, 128, lowIn=True, bf16=True)
    c = mfa.FunctionConstantValues()
    d.setFunctionConstants(c)
    try:
        kd = d.kernelDescriptor(KT.forward)
        assert kd.exp2FmaQuarters == 0 and kd.splitPolicy == (4, 8)
        k = mfa.AttentionKernel(kd)
        assert "exp2" not in k.sourceName() and k.launchCount(c) == 2        # 32 blocks / 4 ranges of >= 4
        cached_before = mfa.AttentionKernel.cached(d, KT.forward)._handle.value

        mfa.setParameterTable(KT.forward, FORWARD_TABLE)
        assert d.parameterFile(KT.forward) == FORWARD_TABLE
        kd = d.kernelDescriptor(KT.forward)
        assert kd.exp2FmaQuarters == 1 and kd.splitPolicy == (2, 16)
        mfa.AttentionKernel(kd)
        assert mfa.AttentionKernel.cached(d, KT.forward)._handle.value != cached_before   # the cache follows the table
        kd64 = make(2048, 2048, 64, lowIn=True).kernelDescriptor(KT.forward)
        assert kd64.exp2FmaQuarters == 2 and kd64.splitPolicy == (8, 4)

        # a table may turn splitting off; the descriptor is plain data and may be edited field by field as well
        kd.splitPolicy = (0, 1)
        assert mfa.AttentionKernel(kd).launchCount(c) == 1
        for q in range(mfa.maxExp2FmaQuarters(KT.forward) + 1):
            kd.exp2FmaQuarters = q
            mfa.AttentionKernel(kd)
        kd.exp2FmaQuarters = mfa.maxExp2FmaQuarters(KT.forward) + 1
        with pytest.raises(mfa.MFAError, match="no compiled sm_90a kernel"):
            mfa.AttentionKernel(kd)

        # rejected tables leave the installed one untouched
        for bad, message in ((FORWARD_TABLE.replace("| 2 | 8 | 4 |", "| 3 | 8 | 4 |"), "no compiled kernel"),
                             (FORWARD_TABLE.replace("Q, O", "Q, dQ", 1), "Unexpected operand: dQ"),
                             ("| 64 | 256 | 128 |\n", "Number of segments was invalid"),
                             ("| 64 | 256 | 128 | 64 | Q, O |\n", "tuning columns")):
            with pytest.raises(mfa.MFAError, match=message):
                mfa.setParameterTable(KT.forward, bad)
            assert d.parameterFile(KT.forward) == FORWARD_TABLE
        # the backward kernels have their own tables and a wider compiled range
        mfa.setParameterTable(KT.backwardQuery, "| 128 | 128 | 64 | 128 | Q, dO, dQ | 3 | 2 | 8 |\n")
        kdq = d.kernelDescriptor(KT.backwardQuery)
        assert kdq.exp2FmaQuarters == 3 and kdq.splitPolicy == (2, 8)
        mfa.AttentionKernel(kdq)
    finally:
        for t in KT:
            mfa.setParameterTable(t, None)
    assert d.kernelDescriptor(KT.forward).exp2FmaQuarters == 0


def test_parameter_file_from_the_environment(tmp_path):
    """MFA_B200_PARAMETER_FILE: tables in that file are picked up when the library is loaded."""
    path = tmp_path / "tables.txt"
    path.write_text("# comment\n[forward]\n" + FORWARD_TABLE + "[backwardKeyValue]\n"
                    "| 64  | 128 | 64  | 64  | K, V, dV, dK | 1 | 2 | 4 |\n| 128 | 128 | 64  | 128 | K, V, dV, dK | 2 | 2 | 8 |\n")
    code = ("import mfa_b200 as mfa\n"
            "d = mfa.AttentionDescriptor(); d.lowPrecisionInputs = True\n"
            "d.matrixDimensions = (512, 512, 64); d.transposeState = (False,) * 4\n"
            "KT = mfa.AttentionKernelType\n"
            "print([(d.kernelDescriptor(t).exp2FmaQuarters,) + d.kernelDescriptor(t).splitPolicy for t in KT])\n")
    out = subprocess.check_output([sys.executable, "-c", code], cwd=ROOT, text=True,
                                  env=dict(os.environ, MFA_B200_PARAMETER_FILE=str(path)))
    assert out.strip() == "[(2, 8, 4), (0, 2, 8), (1, 2, 4)]"   # forward and dK-dV from the file, dQ built in


def test_transposed_tables_are_separate_and_live(tmp_path):
    """Every kernel type has a second table for transposed operands (the layout-generic kernels); run-time replacement
    and the file sections "[....transposed]" reach exactly that table."""
    plain = make(512, 512, 64, lowIn=True)
    trans = make(512, 512, 64, lowIn=True, transposes=(False, True, False, False))
    assert trans.kernelDescriptor(KT.backwardKeyValue).blockDimensions == (128, 64, 64)
    assert plain.kernelDescriptor(KT.backwardKeyValue).blockDimensions == (128, 64, 64)
    try:
        mfa.setParameterTable(KT.backwardKeyValue, "| 256 | 128 | 64 | 256 | K, V, dV, dK | 0 | 4 | 2 |\n", transposed=True)
        assert trans.kernelDescriptor(KT.backwardKeyValue).splitPolicy == (4, 2)
        assert plain.kernelDescriptor(KT.backwardKeyValue).splitPolicy == (2, 8)          # the row-major table is untouched
        with pytest.raises(mfa.MFAError, match="Unexpected operand"):
            mfa.setParameterTable(KT.backwardQuery, "| 256 | 128 | 64 | 256 | K, V | 0 | 2 | 8 |\n", transposed=True)
    finally:
        mfa.setParameterTable(KT.backwardKeyValue, None, transposed=True)
    assert trans.kernelDescriptor(KT.backwardKeyValue).splitPolicy == (2, 8)
    path = tmp_path / "tables.txt"
    path.write_text("[backwardQuery.transposed]\n| 256 | 128 | 64 | 256 | Q, dO, dQ | 0 | 3 | 5 |\n")
    code = ("import mfa_b200 as mfa\n"
            "KT = mfa.AttentionKernelType\n"
            "for t in ((False,) * 4, (True, False, False, False)):\n"
            "    d = mfa.AttentionDescriptor(); d.lowPrecisionInputs = True\n"
            "    d.matrixDimensions = (512, 512, 128); d.transposeState = t\n"
            "    print(d.kernelDescriptor(KT.backwardQuery).splitPolicy)\n")
    out = subprocess.check_output([sys.executable, "-c", code], cwd=ROOT, text=True,
                                  env=dict(os.environ, MFA_B200_PARAMETER_FILE=str(path)))
    assert out.split() == ["(2,", "8)", "(3,", "5)"]


def test_committed_parameter_file_matches_the_builtin_tables():
    """metal-flash-attention_b200/parameters/h100.txt states the built-in defaults: loading it must not change any
    table."""
    path = os.path.join(ROOT, "metal-flash-attention_b200", "parameters", "h100.txt")
    if not os.path.exists(path):
        pytest.skip("no committed sweep result")
    code = ("import mfa_b200 as mfa\n"
            "KT = mfa.AttentionKernelType\n"
            "for D in (64, 128, 256):\n"
            "    d = mfa.AttentionDescriptor(); d.lowPrecisionInputs = True\n"
            "    d.matrixDimensions = (512, 512, D); d.transposeState = (False,) * 4\n"
            "    for t in KT:\n"
            "        kd = d.kernelDescriptor(t)\n"
            "        print(D, int(t), kd.backend.name, kd.blockDimensions, kd.exp2FmaQuarters, kd.splitPolicy)\n")
    plain = subprocess.check_output([sys.executable, "-c", code], cwd=ROOT, text=True,
                                    env={k: v for k, v in os.environ.items() if k != "MFA_B200_PARAMETER_FILE"})
    loaded = subprocess.check_output([sys.executable, "-c", code], cwd=ROOT, text=True,
                                     env=dict(os.environ, MFA_B200_PARAMETER_FILE=path))
    assert plain == loaded
