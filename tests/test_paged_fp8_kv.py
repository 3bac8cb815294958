"""FP8 K/V cache (AttentionKernel.encode(..., paged=, split=, fp8=FP8KV(k_scale, v_scale))): the K and V pools of a
paged forward hold OCP FP8 E4M3 bytes, key row i of K/V head kv standing for k_scale[kv] * e4m3(byte).

The kernels dequantize on load: each byte is converted exactly to Q's 16-bit type in shared memory, and k_scale / v_scale
fold into the softmax scale and the output's normalisation.  So with NULL scales, or powers of two, an FP8 call equals
bit for bit the existing 16-bit paged call (with the same split argument) on the pools dequantized by torch; with
arbitrary scales it meets the paged suite's tolerances against the float64 reference.  NaN bytes outside a sequence's
keys never reach an output, and a captured FP8 split decode replays as the cache grows and the scales change."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import mfa_b200 as mfa
from tests.test_paged_kv import _check_reference, _check_sentinels, build_pool
from tests.test_split_decode import SplitPagedRun, _same
from tests.test_varlen import _constants, _descriptor, _inputs, _offsets, reference
from tests.test_window import band_reference, windowed

KT, Op = mfa.AttentionKernelType, mfa.AttentionOperand
NAN_BYTE = 0x7F


# ------------------------------------------------------------------------------------------------ quantization
def e4m3_bytes(a):
    """float32 array -> its E4M3 bytes (torch's round-to-nearest-even conversion), uint8"""
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def e4m3_values(b):
    """E4M3 bytes -> the values they encode, float32 (exact)"""
    import torch
    return torch.from_numpy(np.ascontiguousarray(b, np.uint8)).view(torch.float8_e4m3fn).to(torch.float32).numpy()


def quantize(x, scales):
    """The E4M3 values (float32) of contiguous keys x [Hkv][T][D] divided by their K/V head's scale"""
    return e4m3_values(e4m3_bytes(x / np.asarray(scales, np.float32)[:, None, None]))


def dequantize(pool, scales):
    """What an FP8 pool [pages][P][Hkv][D] of E4M3 values (rounded to E4M3 first) stands for, float32"""
    return e4m3_values(e4m3_bytes(pool)) * np.asarray(scales, np.float32)[None, None, :, None]


class Fp8PagedRun(SplitPagedRun):
    """A paged forward over FP8 pools: Kp / Vp hold E4M3 values (unscaled; any other value is rounded to E4M3), uploaded
    as bytes; nan_rows: a boolean mask [pages][P] of pool rows whose bytes are replaced by NaN (0x7F); k_scale /
    v_scale: per-K/V-head scales uploaded as device arrays, or None for NULL.  split None: the unsplit FP8 call."""

    def __init__(self, desc, G, Q, Kp, Vp, qo, lengths, table, k_scale=None, v_scale=None, split=None, nan_rows=None):
        import torch
        super().__init__(desc, G, Q, e4m3_values(e4m3_bytes(Kp)), e4m3_values(e4m3_bytes(Vp)), qo, lengths, table,
                         split=split)
        pools = []
        for pool in (Kp, Vp):
            b = e4m3_bytes(pool)
            if nan_rows is not None:
                b[nan_rows] = NAN_BYTE
            pools.append(torch.from_numpy(b).cuda())
        self.k, self.v = pools
        self.scales = [None if s is None else torch.tensor(np.asarray(s, np.float32), device="cuda")
                       for s in (k_scale, v_scale)]
        self.fp8 = mfa.FP8KV(*(0 if s is None else s.data_ptr() for s in self.scales))

    def encode(self, stream=0):
        self.kernel.encode(self.constants, {Op.Q: self.q.data_ptr(), Op.K: self.k.data_ptr(), Op.V: self.v.data_ptr(),
                                            Op.O: self.O.data_ptr(), Op.L: self.L.data_ptr()},
                           stream, paged=self.paged, split=self.split, fp8=self.fp8)


# ------------------------------------------------------------------------------------------------ CPU: the API
def test_fp8_struct_and_version():
    assert ctypes.sizeof(mfa.FP8KV) == 16
    assert {n: getattr(mfa.FP8KV, n).offset for n, _ in mfa.FP8KV._fields_} == {"k_scale": 0, "v_scale": 8}
    assert "FP8 K/V" in mfa.version() and " 0.5 " in mfa.version() and "split-KV decode" in mfa.version()
    assert hasattr(mfa._lib, "mfa_attention_kernel_encode_paged_fp8")


def test_conversion_helpers_are_exact():
    """Every finite E4M3 byte round-trips, and its value is exact in FP16 and BF16 (what the kernels convert to)."""
    import torch
    b = np.arange(256, dtype=np.uint8)
    v = e4m3_values(b)
    finite = np.isfinite(v)
    assert (~finite).sum() == 2 and np.isnan(v[[0x7F, 0xFF]]).all()
    assert np.array_equal(e4m3_bytes(v[finite]), b[finite])
    for dtype in (torch.float16, torch.bfloat16):
        t = torch.from_numpy(v[finite])
        assert torch.equal(t.to(dtype).to(torch.float32), t)


def _paged(S=2, max_row=1, stride=4, page=16):
    return mfa.PagedKV(S, max_row, 16, 16, 16, stride, page)   # (device pointers are not dereferenced on the host)


def _expect_error(call, message):
    with pytest.raises(mfa.MFAError) as e:
        call()
    assert e.value.status == -2 and message in e.value.message, e.value.message


def _raw_encode(kernel, c, paged, split, fp8):
    arr = (ctypes.c_void_p * mfa.MFA_BUFFER_COUNT)()
    return lambda: mfa._check(mfa._lib.mfa_attention_kernel_encode_paged_fp8(
        kernel._handle, ctypes.byref(c._c), ctypes.byref(paged) if paged is not None else None,
        ctypes.byref(split) if split is not None else None, ctypes.byref(fp8) if fp8 is not None else None,
        ctypes.byref(arr), None))


def test_invalid_fp8_requests_are_rejected():
    """Each rejection names its field, before any device work (no GPU is needed to reach them)."""
    desc = _descriptor(256, 128, 64, "bf16", 4, False)
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    c = _constants(256, 128, 4, 2)
    fp8 = mfa.FP8KV()
    _expect_error(_raw_encode(kernel, c, _paged(), None, None), "NULL fp8")
    _expect_error(_raw_encode(kernel, c, _paged(), mfa.SplitKV(), None), "NULL fp8")
    # the paged and split checks come first, made identically
    _expect_error(_raw_encode(kernel, c, None, None, fp8), "NULL paged K/V table")
    for split in (None, mfa.SplitKV()):
        _expect_error(lambda: kernel.encode(c, {}, paged=_paged(S=0), split=split, fp8=fp8), "count 0")
        _expect_error(lambda: kernel.encode(c, {}, paged=_paged(page=24), split=split, fp8=fp8), "page_size 24")
        _expect_error(lambda: kernel.encode(c, {}, paged=_paged(stride=0), split=split, fp8=fp8), "page_stride 0")
    _expect_error(lambda: kernel.encode(c, {}, paged=_paged(), split=mfa.SplitKV(17), fp8=fp8), "num_splits 17")
    # backward kernels: only the forward
    for t in (KT.backwardQuery, KT.backwardKeyValue):
        backward = mfa.AttentionKernel(desc.kernelDescriptor(t))
        for split in (None, mfa.SplitKV()):
            _expect_error(lambda: backward.encode(c, {}, paged=_paged(), split=split, fp8=fp8), "only the forward")
    # the SIMT family
    simt = mfa.AttentionKernel(_descriptor(256, 128, 64, "fp32", 4, False).kernelDescriptor(KT.forward))
    for split in (None, mfa.SplitKV()):
        _expect_error(lambda: simt.encode(c, {}, paged=_paged(), split=split, fp8=fp8),
                      "FP8 K/V needs the tensor-core family")
    # head dimensions that are a multiple of 8 but not of 16
    for D in (72, 120):
        k = mfa.AttentionKernel(_descriptor(256, 128, D, "bf16", 4, False).kernelDescriptor(KT.forward))
        _expect_error(lambda: k.encode(c, {}, paged=_paged(), fp8=fp8), f"multiple of 16 (head {D})")
    # the Python mirror: fp8= belongs to paged calls
    _expect_error(lambda: kernel.encode(c, {}, fp8=fp8), "fp8= needs paged=")
    _expect_error(lambda: kernel.encode(c, {}, sequences=mfa.SequenceTable(2, 10, 10, 16, 16), fp8=fp8),
                  "fp8= needs paged=")
    _expect_error(lambda: kernel.encode(c, {}, sequences=mfa.SequenceTable(2, 10, 10, 16, 16),
                                        split=mfa.SplitKV(), fp8=fp8), "fp8= needs paged=")


def test_cpp_host_mirror_with_fp8_kv(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  AttentionDescriptor d;
  d.lowPrecisionInputs = false;
  d.matrixDimensions = MatrixDimensions{300, 4096, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.batchCount = 32;
  mfa_function_constants_t constants;
  d.setFunctionConstants(constants);
  kvGroup(constants) = 8;
  static int32_t fake[3];
  PagedKV paged{1, 1, fake, fake, fake, 256, 16};
  const SplitKV split{0, 0};
  const FP8KV fp8{nullptr, nullptr};
  AttentionKernel f(d.kernelDescriptor(AttentionKernelType::forward));   // FP32: the SIMT family
  std::array<void *, MFA_BUFFER_COUNT> buffers{};
  for (const SplitKV *s : {static_cast<const SplitKV *>(nullptr), &split}) {
    try {
      f.encode(constants, paged, s, fp8, buffers);
    } catch (const std::exception &e) {
      std::printf("%s\n", std::strstr(e.what(), "tensor-core family") ? "rejected" : e.what());
    }
  }
  std::printf("%zu\n", sizeof(FP8KV));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-include", "cstring", "-I", root, str(src), "-o", str(exe), "-L",
                           libdir, "-lmfa_b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    assert out[:3] == ["rejected", "rejected", "16"], out


def test_ptxas_fp8_kernels_have_no_spills_and_no_stack_frame():
    from tests.test_forward_pipeline import _ptxas_report
    report, text = _ptxas_report()
    kernels = {name: r for name, r in report.items() if "fp8_kv_" in name}
    # 3 head-dimension chunk counts x bf16 / fp16 Q x (causal or not, or a window)
    assert len(kernels) == 3 * 2 * 3, sorted(kernels)
    for name, r in kernels.items():
        assert r == (0, 0, 0), (name, r)
        assert not re.search(r"C7510.*" + re.escape(name), text), name
        # (the existing suites count their kernels by these names)
        assert "split_forward_" not in name and "paged_forward_wgmma" not in name, name
        assert not re.search(r"attention_\w+_wgmma|band_\w+_wgmma", name), name


# ------------------------------------------------------------------------------------------------ GPU
# Each GPU check runs in a process of its own, and this file sorts after tests/test_host_api.py.  The host API suite's
# launch-count test records one encode with torch.profiler and no warm-up kernel inside the profiled window.  On an
# H100 it passed at the parent commit (whole GPU suite), on its own, after the causal suite alone, and after these
# checks alone; it recorded too few kernels, or none, whenever these checks ran between the causal suite's profiler
# session and it -- in the pytest process, and also from subprocesses.  Run in the pytest process before the split
# suite, these checks also once made that suite's trace test miss a kernel.  Which state carries over was not found:
# the existing traces are fragile to what runs before them, and these checks stay out of their way.
def _isolated(check, *args):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); from tests import test_paged_fp8_kv as t; "
            f"t.{check}(*{args!r})")
    proc = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]


LENGTHS = {  # (query lengths Rs, key lengths Cs)
    # decode rows (one head-packed tile per K/V head), a sequence without keys, and causal Rs > Cs
    "decode": ([1, 1, 1, 1, 2, 1], [0, 1, 40, 300, 1, 1500]),
    # chunk rows (Rs > 128, two tiles), a sequence without keys, and causal Rs > Cs
    "chunk": ([200, 1, 130, 3], [700, 0, 300, 2]),
}
# a pairwise selection over (mode, D, causal, G, page size, window, lengths); every case runs split None, 1, plan and 4
MATRIX = [
    ("bf16", 64, True, 1, 16, None, "decode"),
    ("bf16", 80, False, 4, 64, (100, 20), "chunk"),
    ("bf16", 128, True, 8, 256, (63, 0), "decode"),
    ("bf16", 256, False, 4, 16, None, "decode"),
    ("bf16", 128, False, 1, 64, None, "chunk"),
    ("bf16", 256, True, 8, 64, (63, 0), "chunk"),
    ("reference", 64, False, 8, 256, (100, 20), "decode"),
    ("reference", 80, True, 8, 16, None, "decode"),
    ("reference", 128, True, 4, 16, (63, 0), "chunk"),
    ("reference", 256, True, 1, 256, None, "chunk"),
    ("reference", 64, True, 4, 64, (63, 0), "chunk"),
    ("reference", 128, False, 1, 256, (100, 20), "decode"),
    ("bf16", 80, True, 1, 256, (63, 0), "decode"),
    ("reference", 80, False, 1, 64, None, "chunk"),
]
SPLITS = {"None": None, "1": (1,), "plan": (), "4": (4,)}


def _case(mode, D, causal, G, page_size, lengths, seed, k_scale=None, v_scale=None):
    """Descriptor, inputs (K, V replaced by their scaled E4M3 values), offsets, key lengths, and the E4M3-valued
    pools and table (k_scale / v_scale: per-K/V-head, default 1)."""
    rq, rk = LENGTHS[lengths]
    qo, ko = _offsets(rq), _offsets(rk)
    H = 8
    T, Tk = qo[-1] + 9, ko[-1] + 5   # query rows past the table's end keep their sentinels
    desc = _descriptor(T, Tk, D, mode, H, causal)
    x = _inputs(desc, G, T, Tk, seed)
    sk, sv = (np.ones(H // G, np.float32) if s is None else np.asarray(s, np.float32) for s in (k_scale, v_scale))
    Kq, Vq = quantize(x[Op.K], sk), quantize(x[Op.V], sv)
    Kp, Vp, table = build_pool(Kq, Vq, ko, page_size, np.random.default_rng(seed))
    x = {**x, Op.K: Kq * sk[:, None, None], Op.V: Vq * sv[:, None, None], Op.dO: np.zeros_like(x[Op.Q])}
    return desc, x, qo, ko, rk, Kp, Vp, table


def _reference(x, G, qo, ko, causal, window):
    if window is None:
        return reference(x, G, qo, ko, causal)
    return band_reference(x, G, qo, ko, window[0], 0 if causal else window[1])


def _window(window):
    import contextlib
    return windowed(window) if window else contextlib.nullcontext()


def _run(run):
    run.encode()
    return run.results()


def _pow2_scales(G, seed):
    """Power-of-two scales for K and V, one per K/V head, every V scale different from its head's K scale (and the V
    scales in the reverse head order), so that a swapped or shared scale pointer cannot give the same bits"""
    k = (2.0 ** np.random.default_rng(seed).integers(-6, -2, 8 // G)).astype(np.float32)
    return k, (2 * k)[::-1].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("scaled", [False, True], ids=["null_scales", "pow2_scales"])
@pytest.mark.parametrize("mode,D,causal,G,page_size,window,lengths", MATRIX)
def test_fp8_equals_the_16bit_call_on_dequantized_pools(mode, D, causal, G, page_size, window, lengths, scaled):
    """NULL scales, or a different power of two per K/V head: O and L equal the 16-bit paged call on the pools
    dequantized by torch, bit for bit, for split None, SplitKV(1), SplitKV() and SplitKV(4)."""
    _isolated("_check_bitwise", mode, D, causal, G, page_size, window, lengths, scaled)


def _check_bitwise(mode, D, causal, G, page_size, window, lengths, scaled):
    seed = D + G + page_size + scaled
    sk, sv = _pow2_scales(G, seed) if scaled else (None, None)
    desc, x, qo, ko, rk, Kp, Vp, table = _case(mode, D, causal, G, page_size, lengths, seed, sk, sv)
    ones = np.ones(8 // G, np.float32)
    with _window(window):
        for name, split in SPLITS.items():
            split = None if split is None else mfa.SplitKV(*split)
            fp8 = _run(Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, sk, sv, split=split))
            plain = _run(SplitPagedRun(desc, G, x[Op.Q], dequantize(Kp, ones if sk is None else sk),
                                       dequantize(Vp, ones if sv is None else sv), qo, rk, table, split=split))
            _same(fp8, plain)
            _check_sentinels(fp8, qo)
    _check_reference(fp8, _reference(x, G, qo, ko, causal, window), qo, "fp16" if mode == "reference" else mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,G,window,lengths", [
    ("bf16", 128, True, 4, None, "decode"), ("reference", 64, False, 8, (100, 20), "chunk"),
    ("bf16", 256, True, 1, (63, 0), "chunk"), ("reference", 80, True, 4, None, "decode")])
def test_fp8_with_arbitrary_scales_meets_the_reference(mode, D, causal, G, window, lengths):
    """Per-head scales from each head's absolute maximum (as a serving engine calibrates them), K and V different: the
    paged suite's tolerances against the float64 reference on the dequantized values, for each split argument."""
    _isolated("_check_arbitrary_scales", mode, D, causal, G, window, lengths)


def _check_arbitrary_scales(mode, D, causal, G, window, lengths):
    rng = np.random.default_rng(D + G)
    rq, rk = LENGTHS[lengths]
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 9, ko[-1] + 5
    desc = _descriptor(T, Tk, D, mode, 8, causal)
    x = _inputs(desc, G, T, Tk, seed=D)
    # (the head's absolute maximum maps to 400 or less, inside E4M3's 448)
    k_scale, v_scale = (np.abs(x[op]).max(axis=(1, 2)).astype(np.float32) / 400 * rng.uniform(1.0, 1.5, 8 // G)
                        for op in (Op.K, Op.V))
    k_scale, v_scale = k_scale.astype(np.float32), v_scale.astype(np.float32)
    Kq, Vq = quantize(x[Op.K], k_scale), quantize(x[Op.V], v_scale)
    Kp, Vp, table = build_pool(Kq, Vq, ko, 64, np.random.default_rng(D))
    ref_inputs = {Op.Q: x[Op.Q], Op.K: Kq * k_scale[:, None, None], Op.V: Vq * v_scale[:, None, None],
                  Op.dO: np.zeros_like(x[Op.Q])}
    with _window(window):
        ref = _reference(ref_inputs, G, qo, ko, causal, window)
        for split in (None, mfa.SplitKV(1), mfa.SplitKV(), mfa.SplitKV(4)):
            out = _run(Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, k_scale, v_scale, split=split))
            _check_sentinels(out, qo)
            _check_reference(out, ref, qo, "fp16" if mode == "reference" else mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,window", [("bf16", None), ("reference", None), ("bf16", (63, 0))])
def test_nan_bytes_outside_the_keys_never_reach_an_output(mode, window):
    """0x7F (NaN) in every pool row past each Cs and in spare pages, page-table entries past a sequence's last page
    at -1 or a huge id, and (window) the pages wholly before the band pointing at a NaN page: O and L equal the run
    with finite filler bit for bit."""
    _isolated("_check_nan_bytes", mode, window)


def _check_nan_bytes(mode, window):
    rq, rk = [1, 2, 1, 0, 100], [40, 0, 3000, 40, 700]
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 9, ko[-1] + 5
    G, P = 4, 16
    desc = _descriptor(T, Tk, 128, mode, 8, True)
    x = _inputs(desc, G, T, Tk, seed=6)
    k_scale, v_scale = _pow2_scales(G, 6)
    Kq, Vq = quantize(x[Op.K], k_scale), quantize(x[Op.V], v_scale)
    Kp, Vp, table = build_pool(Kq, Vq, ko, P, np.random.default_rng(6))
    # the pool rows that hold a key of some sequence
    used = np.zeros(Kp.shape[:2], bool)
    for s, Cs in enumerate(rk):
        for i in range(Cs):
            used[table[s, i // P], i % P] = True
    with _window(window):
        for split in (None, mfa.SplitKV(), mfa.SplitKV(16)):
            clean = _run(Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, k_scale, v_scale, split=split))
            for tail in (-1, 2**31 - 1):
                dirty_table = table.copy()
                for s, Cs in enumerate(rk):
                    dirty_table[s, -(-Cs // P):] = tail
                    if window is not None and rq[s]:
                        first = (Cs - rq[s] - window[0]) // P   # pages wholly before the band of the first query row
                        nan_page = int(np.flatnonzero(~used.any(axis=1))[0])   # a spare page: all NaN
                        dirty_table[s, :max(first, 0)] = nan_page
                dirty = _run(Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, dirty_table, k_scale, v_scale, split=split,
                                         nan_rows=~used))
                _check_sentinels(dirty, qo)
                _same(clean, dirty)
    ref = _reference({**x, Op.K: Kq * k_scale[:, None, None], Op.V: Vq * v_scale[:, None, None],
                      Op.dO: np.zeros_like(x[Op.Q])}, G, qo, ko, True, window)
    _check_reference(clean, ref, qo, "fp16" if mode == "reference" else mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "reference"])
def test_fp8_split_decode_replays_in_a_cuda_graph(mode):
    """A captured FP8 split decode (library plan, long context) replayed after column_lengths and page_table grew by a
    token and the scales were rewritten in place equals an eager encode bit for bit; two eager runs agree."""
    _isolated("_check_graph_replay", mode)


def _check_graph_replay(mode):
    import torch
    P, G, H, D = 16, 4, 8, 128
    before = [2047, 15]
    after = [c + 1 for c in before]
    qo = _offsets([1] * len(before))
    T = qo[-1]
    desc = _descriptor(T, 4096, D, mode, H, True)
    rng = np.random.default_rng(31)
    x = _inputs(desc, G, T, sum(after), seed=31)
    ko_after = _offsets(after)
    s0 = np.full(H // G, 2.0 ** -4, np.float32)
    k1, v1 = np.array([0.011, 0.023], np.float32), np.array([0.019, 0.013], np.float32)   # (K and V differ)
    Kq, Vq = quantize(x[Op.K], k1), quantize(x[Op.V], v1)
    Kp, Vp, table_after = build_pool(Kq, Vq, ko_after, P, rng, spare_pages=8)
    table_before = table_after.copy()
    for s, c in enumerate(before):
        table_before[s, -(-c // P):] = -1
    run = Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, before, table_before, s0, s0, split=mfa.SplitKV())
    assert run.plan().splits > 1
    stream = torch.cuda.Stream()
    run.encode(stream.cuda_stream)   # (outside any capture first, on the capturing stream: its workspace)
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        run.encode(stream.cuda_stream)
    run.lengths.copy_(torch.tensor(after, dtype=torch.int32))
    run.table.copy_(torch.tensor(table_after, dtype=torch.int32))
    for dev, new in zip(run.scales, (k1, v1)):
        dev.copy_(torch.from_numpy(new))
    run.O.fill_(float("nan"))
    run.L.fill_(float("nan"))
    graph.replay()
    replayed = run.results()
    eager = Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, after, table_after, k1, v1, split=mfa.SplitKV())
    fresh = _run(eager)
    again = _run(eager)
    _same(replayed, fresh)
    _same(fresh, again)
    ref = reference({Op.Q: x[Op.Q], Op.K: Kq * k1[:, None, None], Op.V: Vq * v1[:, None, None],
                     Op.dO: np.zeros_like(x[Op.Q])}, G, qo, ko_after, True)
    _check_reference(replayed, ref, qo, "fp16" if mode == "reference" else mode)
