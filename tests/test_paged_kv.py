"""Paged K/V cache (AttentionKernel.encode(..., paged=PagedKV)): the forward reads K and V through a per-sequence page
table, in place, from pools [num_pages][P][Hkv][D] (vLLM's block table).

Queries, O and L keep the packed layout of tests/test_varlen.py ([H][row][D], [H][row], sequence s owns rows
[qo[s], qo[s + 1])).  Sequence s has Cs keys; key i is pool row page_table[s][i // P] * P + i % P.  Paging only changes
where the rows of a key block come from, so on the GPU a paged call must equal bit for bit the packed call on the same
keys laid out contiguously; it must also meet the packed suite's tolerances against the float64 reference, ignore
whatever the pool holds outside a sequence's keys (NaN included) and page-table entries past its last page, leave rows
outside every sequence untouched, and replay from a CUDA graph after the cache grew by a token."""
import ctypes

import numpy as np
import pytest

import mfa_b200 as mfa
import oracle
from tests.test_varlen import LOG2E, _constants, _descriptor, _inputs, _offsets, reference

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision


# ------------------------------------------------------------------------------------------------ the page pools
def build_pool(K, V, ko, page_size, rng, spare_pages=3, fill=None, tail=None):
    """Scatters the contiguous keys of every sequence (K, V [Hkv][Tk][D], sequence s in rows [ko[s], ko[s + 1])) into
    shuffled pages of pools [num_pages][page_size][Hkv][D], with `spare_pages` pages that no sequence owns.  fill: the
    value of every pool row no key occupies (default: random finite values).  tail: page-table entries past a
    sequence's last page (default: random pages of the pool).  Returns (K pool, V pool, page_table [S][stride])."""
    Hkv, _, D = K.shape
    lengths = np.diff(ko)
    pages_of = [-(-int(c) // page_size) for c in lengths]
    stride = max(1, max(pages_of) + 1)
    num_pages = sum(pages_of) + spare_pages
    order = rng.permutation(num_pages)
    pools = []
    for src in (K, V):
        pool = (rng.standard_normal((num_pages, page_size, Hkv, D)) if fill is None else
                np.full((num_pages, page_size, Hkv, D), fill))
        pools.append(pool.astype(np.float32))
    table = rng.integers(0, num_pages, (len(lengths), stride)) if tail is None else np.full((len(lengths), stride), tail)
    table = table.astype(np.int64)
    n = 0
    for s, count in enumerate(pages_of):
        for j in range(count):
            page = int(order[n])
            n += 1
            table[s, j] = page
            rows = slice(ko[s] + j * page_size, min(ko[s + 1], ko[s] + (j + 1) * page_size))
            used = rows.stop - rows.start
            for pool, src in zip(pools, (K, V)):
                pool[page, :used] = np.swapaxes(src[:, rows], 0, 1)
    return pools[0], pools[1], table


def gather(pool, table, lengths, page_size):
    """The keys of every sequence read back through the page table, contiguous: [Hkv][sum(lengths)][D]."""
    parts = []
    for s, count in enumerate(lengths):
        rows = [pool[table[s, i // page_size], i % page_size] for i in range(int(count))]
        parts.append(np.stack(rows) if rows else np.zeros((0,) + pool.shape[2:], pool.dtype))
    return np.swapaxes(np.concatenate(parts), 0, 1)


# ------------------------------------------------------------------------------------------------ CPU: the API
def _paged(S=2, max_row=10, rows=16, lengths=16, table=16, stride=4, page=16):
    return mfa.PagedKV(S, max_row, rows, lengths, table, stride, page)


def test_paged_kv_layout_and_version():
    assert ctypes.sizeof(mfa.PagedKV) == 40
    offsets = {name: getattr(mfa.PagedKV, name).offset for name, _ in mfa.PagedKV._fields_}
    assert offsets == {"count": 0, "max_row": 4, "row_offsets": 8, "column_lengths": 16, "page_table": 24,
                       "page_stride": 32, "page_size": 36}
    assert "paged K/V" in mfa.version() and " 0.5 " in mfa.version()


def test_grid_size_and_launch_count_of_paged_calls():
    """Grid (tiles of the longest query sequence, heads, S), one launch, for the tensor-core and SIMT families."""
    H, G = 8, 4
    for mode in ("bf16", "reference", "fp32"):
        desc = _descriptor(4096, 4096, 128, mode, H, True)
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
        par = kernel.blockDimensions[0]
        c = _constants(4096, 64 * 256, H, G)
        for S, max_row in ((1, 1), (64, 1), (3, 1000), (8, 4096)):
            paged = _paged(S=S, max_row=max_row, page=256)
            assert kernel.gridSize(c, paged=paged) == -(-max_row // par) * H * S, (mode, S)
            assert kernel.launchCount(c, paged=paged) == 1


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_invalid_paged_tables_are_rejected(mode):
    desc = _descriptor(256, 128, 64, mode, 4, False)
    c = _constants(256, 128, 4, 2)
    bad = [(None, "NULL paged K/V table"),
           (_paged(rows=0), "row_offsets must not be NULL"),
           (_paged(lengths=0), "column_lengths must not be NULL"),
           (_paged(table=0), "page_table must not be NULL"),
           (_paged(S=0), "count 0"),
           (_paged(S=65536), "count 65536"),
           (_paged(max_row=0), "max_row 0"),
           (_paged(max_row=257), "max_row 257"),
           (_paged(page=8), "page_size 8"),
           (_paged(page=48), "page_size 48"),
           (_paged(page=256), "page_size 256"),     # does not divide column = 128
           (_paged(page=0), "page_size 0"),
           (_paged(stride=0), "page_stride 0")]
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    for table, message in bad:
        for name in ("grid_size", "launch_count"):
            with pytest.raises(mfa.MFAError) as e:
                if table is None:
                    out = ctypes.c_uint32()
                    fn = getattr(mfa._lib, f"mfa_attention_kernel_{name}_paged")
                    mfa._check(fn(kernel._handle, ctypes.byref(c._c), None, ctypes.byref(out)))
                else:
                    (kernel.gridSize if name == "grid_size" else kernel.launchCount)(c, paged=table)
            assert e.value.status == -2 and message in e.value.message, (table, e.value.message)
    # backward kernels, a batch of more than one launch slice
    for t in (KT.backwardQuery, KT.backwardKeyValue):
        backward = mfa.AttentionKernel(desc.kernelDescriptor(t))
        for call in (backward.gridSize, backward.launchCount):
            with pytest.raises(mfa.MFAError) as e:
                call(c, paged=_paged())
            assert e.value.status == -2 and "only the forward" in e.value.message
    big = _descriptor(256, 128, 64, mode, 16385, False)
    kernel = mfa.AttentionKernel(big.kernelDescriptor(KT.forward))
    for call in (kernel.gridSize, kernel.launchCount):
        with pytest.raises(mfa.MFAError) as e:
            call(_constants(256, 128, 16385, 1), paged=_paged())
        assert e.value.status == -2 and "batch_count 16385" in e.value.message


@pytest.mark.parametrize("mode,D,transpose,message", [
    ("bf16", 128, (False, True, False, False), "K is transposed"),
    ("fp32", 64, (True, False, False, False), "Q is transposed"),
    ("bf16", 60, (False,) * 4, "multiple of 8"),
])
def test_paged_calls_need_row_major_operands_and_tensor_core_heads(mode, D, transpose, message):
    desc = _descriptor(256, 128, D, mode, 4, False, transpose)
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    c = _constants(256, 128, 4, 2)
    assert kernel.gridSize(c) > 0   # fixed-length calls take these descriptors
    for call in (kernel.gridSize, kernel.launchCount):
        with pytest.raises(mfa.MFAError) as e:
            call(c, paged=_paged())
        assert e.value.status == -2 and message in e.value.message, e.value.message


def test_sequences_and_paged_are_exclusive():
    desc = _descriptor(256, 128, 64, "bf16", 4, False)
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    c = _constants(256, 128, 4, 2)
    table = mfa.SequenceTable(2, 10, 10, 16, 16)
    for call in (kernel.gridSize, kernel.launchCount, lambda c, **kw: kernel.encode(c, {}, **kw)):
        with pytest.raises(mfa.MFAError) as e:
            call(c, sequences=table, paged=_paged())
        assert "not both" in e.value.message


def test_cpp_host_mirror_with_paged_kv(tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  AttentionDescriptor d;
  d.lowPrecisionInputs = true;
  d.matrixDimensions = MatrixDimensions{300, 4096, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  d.batchCount = 32;
  mfa_function_constants_t constants;
  d.setFunctionConstants(constants);
  kvGroup(constants) = 8;
  static int32_t fake[3];
  PagedKV paged{64, 1, fake, fake, fake, 256, 16};
  AttentionKernel f(d.kernelDescriptor(AttentionKernelType::forward));
  std::printf("%u %u %zu\n", f.gridSize(constants, paged), f.launchCount(constants, paged), sizeof(mfa_paged_kv_t));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", root, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert out == [str(32 * 64), "1", str(ctypes.sizeof(mfa.PagedKV))], out


@pytest.mark.parametrize("page_size", [16, 64, 256])
def test_pool_builder_round_trips(page_size):
    """Scattering contiguous K/V into shuffled pages and gathering them back through the table is the identity, and
    the pages of different sequences are distinct."""
    rng = np.random.default_rng(page_size)
    lengths = [1, 0, 63, 64, 65, 300, 16]
    ko = _offsets(lengths)
    K, V = (rng.standard_normal((3, ko[-1], 8)).astype(np.float32) for _ in range(2))
    Kp, Vp, table = build_pool(K, V, ko, page_size, rng)
    assert Kp.shape[1:] == (page_size, 3, 8)
    assert np.array_equal(gather(Kp, table, lengths, page_size), K)
    assert np.array_equal(gather(Vp, table, lengths, page_size), V)
    used = [table[s, j] for s, c in enumerate(lengths) for j in range(-(-c // page_size))]
    assert len(set(used)) == len(used) and len(used) + 3 == Kp.shape[0]


def test_ptxas_paged_tensor_core_kernels_have_no_spills_and_no_stack_frame():
    import re
    from tests.test_forward_pipeline import _ptxas_report
    report, text = _ptxas_report()
    kernels = {name: r for name, r in report.items() if "paged_forward_wgmma" in name}
    assert len(kernels) == 12, sorted(kernels)   # 3 head-dimension chunk counts x bf16 / fp16 x causal or not
    for name, r in kernels.items():
        assert not re.search(r"attention_\w+_wgmma", name), name
        assert r == (0, 0, 0), (name, r)
        assert not re.search(r"C7510.*" + re.escape(name), text), name


# ------------------------------------------------------------------------------------------------ GPU
def _upload(a, prec):
    """float32 array (already representable in prec) -> device tensor holding its memory image"""
    import torch
    raw = oracle.encode(np.ascontiguousarray(a, np.float32), int(prec))
    return torch.from_numpy(raw.view(np.int16) if prec != P.FP32 else raw).cuda()


def _outputs(H, T, D, prec_L=P.FP32):
    """NaN-sentinel O (FP32) and L (FP32, or 0xFFFF -- NaN -- in a 16-bit L)."""
    import torch
    L = (torch.full((H * T,), float("nan"), device="cuda") if prec_L == P.FP32 else
         torch.full((H * T,), -1, dtype=torch.int16, device="cuda"))
    return torch.full((H * T * D,), float("nan"), device="cuda"), L


def _download_L(L, prec_L, H, T):
    """L as float32 [H][T] (decoded from a 16-bit L)"""
    a = L.cpu().numpy()
    return (a if prec_L == P.FP32 else oracle.decode(a.view(np.uint16), int(prec_L))).reshape(H, T)


def run_packed_forward(desc, G, Q, K, V, qo, ko):
    """The packed forward over contiguous keys: {O: [H][T][D], L: [H][T]} float32 (raw, L in log2 units)."""
    import torch
    prec = desc.memoryPrecisions
    assert prec[Op.O] == P.FP32
    H, T, D = Q.shape
    q, k, v = _upload(Q, prec[Op.Q]), _upload(K, prec[Op.K]), _upload(V, prec[Op.V])
    O, L = _outputs(H, T, D, prec[Op.L])
    tq, tk = (torch.tensor(x, dtype=torch.int32, device="cuda") for x in (qo, ko))
    rq, rk = np.diff(qo), np.diff(ko)
    table = mfa.SequenceTable(len(qo) - 1, max(1, int(rq.max())), max(1, int(rk.max())), tq.data_ptr(), tk.data_ptr())
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    kernel.encode(_constants(T, K.shape[1], H, G),
                  {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(), Op.L: L.data_ptr()},
                  sequences=table)
    torch.cuda.synchronize()
    return {"O": O.cpu().numpy().reshape(H, T, D), "L": _download_L(L, prec[Op.L], H, T)}


class PagedRun:
    """Device buffers of one paged forward: Q, the pools, the three tables and NaN-sentinel outputs."""

    def __init__(self, desc, G, Q, Kp, Vp, qo, lengths, table, max_row=None):
        import torch
        prec = desc.memoryPrecisions
        self.H, self.T, self.D = Q.shape
        self.page_size = Kp.shape[1]
        self.q, self.k, self.v = _upload(Q, prec[Op.Q]), _upload(Kp, prec[Op.K]), _upload(Vp, prec[Op.V])
        self.prec_L = prec[Op.L]
        self.O, self.L = _outputs(self.H, self.T, self.D, self.prec_L)
        self.rows = torch.tensor(qo, dtype=torch.int32, device="cuda")
        self.lengths = torch.tensor(np.asarray(lengths, np.int64), dtype=torch.int32, device="cuda")
        self.table = torch.tensor(np.clip(table, -2**31, 2**31 - 1), dtype=torch.int32, device="cuda")
        self.paged = mfa.PagedKV(len(qo) - 1, max_row or max(1, int(np.diff(qo).max())), self.rows.data_ptr(),
                                 self.lengths.data_ptr(), self.table.data_ptr(), table.shape[1], self.page_size)
        self.constants = _constants(self.T, Kp.shape[0] * self.page_size, self.H, G)
        self.kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))

    def encode(self, stream=0):
        self.kernel.encode(self.constants, {Op.Q: self.q.data_ptr(), Op.K: self.k.data_ptr(), Op.V: self.v.data_ptr(),
                                            Op.O: self.O.data_ptr(), Op.L: self.L.data_ptr()},
                           stream, paged=self.paged)

    def results(self):
        import torch
        torch.cuda.synchronize()
        return {"O": self.O.cpu().numpy().reshape(self.H, self.T, self.D),
                "L": _download_L(self.L, self.prec_L, self.H, self.T)}


def run_paged_forward(desc, G, Q, Kp, Vp, qo, lengths, table):
    run = PagedRun(desc, G, Q, Kp, Vp, qo, lengths, table)
    run.encode()
    return run.results()


def _check_reference(out, ref, qo, mode):
    """The packed suite's forward tolerances against the float64 reference (rows inside the sequences)."""
    T = qo[-1]
    O, L = out["O"][:, :T], out["L"][:, :T] / np.float32(LOG2E)
    rO, rL = ref["O"][:, :T], ref["L"][:, :T].copy()
    inf = np.isposinf(rL)
    assert (np.isposinf(L) == inf).all(), "rows that see no key get L = +inf"
    L = np.where(inf, 0.0, L)
    rL[inf] = 0.0
    assert np.isfinite(O).all() and np.isfinite(L).all()
    fp32 = mode == "fp32"
    bars = {"O": 2e-5 if fp32 else (2e-2 if mode == "bf16" else 5e-3), "L": 2e-5 if fp32 else 1e-3}
    for name, got, want in (("O", O, rO), ("L", L, rL)):
        err = float(np.abs(got - want).max())
        assert err <= bars[name], f"{name}: {err:.3e} > {bars[name]}"


def _check_sentinels(out, qo):
    assert np.isnan(out["O"][:, qo[-1]:]).all() and np.isnan(out["L"][:, qo[-1]:]).all()


LENGTHS = {  # (query lengths Rs, key lengths Cs)
    "edges": ([1, 63, 64, 65, 127, 129, 1000], [1, 63, 64, 65, 127, 129, 1000]),
    "decode": ([1, 1, 1, 1, 1, 100], [1, 64, 65, 129, 1000, 3000]),   # decode rows and a chunked-prefill row
    "empty": ([70, 0, 130, 200, 1], [90, 50, 0, 100, 127]),            # Rs = 0, Cs = 0, Rs > Cs
}
CASES = [  # (mode, D, causal, G, page size, lengths)
    ("bf16", 128, True, 4, 16, "edges"), ("bf16", 128, False, 1, 256, "decode"), ("bf16", 64, True, 1, 32, "empty"),
    ("fp16", 64, False, 4, 64, "edges"), ("fp16", 256, True, 4, 128, "decode"), ("bf16", 256, False, 1, 16, "empty"),
    ("reference", 128, True, 4, 64, "empty"), ("reference", 64, False, 1, 128, "decode"),
    ("bf16", 72, True, 4, 256, "edges"), ("fp16", 72, True, 1, 16, "decode"), ("bf16", 64, True, 4, 16, "decode"),
    ("bf16", 128, True, 4, 128, "decode"), ("fp32", 72, True, 4, 16, "empty"), ("fp32", 320, False, 1, 64, "decode"),
]


def _case(mode, D, causal, G, lengths, seed):
    rq, rk = LENGTHS[lengths]
    qo, ko = _offsets(rq), _offsets(rk)
    H = 4
    T, Tk = qo[-1] + 9, ko[-1] + 5   # query rows past the table's end keep their sentinels
    desc = _descriptor(T, Tk, D, mode, H, causal)
    return desc, _inputs(desc, G, T, Tk, seed), qo, ko, rk


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,G,page_size,lengths", CASES)
def test_paged_equals_packed_bitwise_and_meets_the_reference(mode, D, causal, G, page_size, lengths):
    desc, inputs, qo, ko, rk = _case(mode, D, causal, G, lengths, seed=D + G + page_size)
    rng = np.random.default_rng(page_size)
    Kp, Vp, table = build_pool(inputs[Op.K], inputs[Op.V], ko, page_size, rng)
    paged = run_paged_forward(desc, G, inputs[Op.Q], Kp, Vp, qo, rk, table)
    packed = run_packed_forward(desc, G, inputs[Op.Q], inputs[Op.K], inputs[Op.V], qo, ko)
    _check_sentinels(paged, qo)
    for name in ("O", "L"):
        assert paged[name].tobytes() == packed[name].tobytes(), name
    _check_reference(paged, reference(inputs, G, qo, ko, causal), qo, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,page_size", [("bf16", 16), ("bf16", 256), ("reference", 64), ("fp32", 32)])
def test_pool_contents_outside_the_sequences_do_not_leak(mode, page_size):
    """NaN / Inf in every pool row no key occupies (spare pages and the tail of each sequence's last page), and
    page-table entries past ceil(Cs / P) of -1 or a huge id: the outputs stay bitwise those of a clean pool."""
    desc, inputs, qo, ko, rk = _case(mode, 128, True, 2, "edges", seed=3)
    Kp, Vp, table = build_pool(inputs[Op.K], inputs[Op.V], ko, page_size, np.random.default_rng(page_size))
    clean = run_paged_forward(desc, 2, inputs[Op.Q], Kp, Vp, qo, rk, table)
    for fill, tail in ((np.nan, -1), (np.inf, 2**31 - 1)):
        Kp, Vp, table = build_pool(inputs[Op.K], inputs[Op.V], ko, page_size, np.random.default_rng(page_size),
                                   fill=fill, tail=tail)
        dirty = run_paged_forward(desc, 2, inputs[Op.Q], Kp, Vp, qo, rk, table)
        _check_sentinels(dirty, qo)
        for name in ("O", "L"):
            assert clean[name].tobytes() == dirty[name].tobytes(), (fill, name)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_paged_encode_replays_in_a_cuda_graph_as_the_cache_grows(mode):
    """A serving loop: one decode encode captured into a CUDA graph, replayed after every sequence's cache grew by one
    token (column_lengths + 1, its K/V written into the pool, and a new page where the length crosses a page boundary).
    The replay equals an eager call on the new contents."""
    import torch
    page_size, G, H, D = 16, 4, 8, 128
    before = [15, 16, 40, 200]          # 15 -> 16 fills a page; 16 -> 17 needs a new one
    after = [c + 1 for c in before]
    qo = _offsets([1] * len(before))
    T = qo[-1]
    desc = _descriptor(T, 512, D, mode, H, True)
    prec = desc.memoryPrecisions
    rng = np.random.default_rng(21)
    x = {op: oracle.roundtrip(rng.standard_normal(shape).astype(np.float32), int(prec[op]))
         for op, shape in ((Op.Q, (H, T, D)), (Op.K, (H // G, sum(after), D)), (Op.V, (H // G, sum(after), D)))}
    ko_after = _offsets(after)
    # the grown cache's pool and table; the table before the step lacks the pages of the new tokens
    Kp, Vp, table_after = build_pool(x[Op.K], x[Op.V], ko_after, page_size, rng, spare_pages=8)
    table_before = table_after.copy()
    for s, c in enumerate(before):
        table_before[s, -(-c // page_size):] = -1
    run = PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, before, table_before)
    run.encode()   # (outside any capture first)
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        run.encode(stream.cuda_stream)
    run.lengths.copy_(torch.tensor(after, dtype=torch.int32))
    run.table.copy_(torch.tensor(table_after, dtype=torch.int32))
    run.O.fill_(float("nan"))
    run.L.fill_(float("nan"))
    graph.replay()
    replayed = run.results()
    eager = run_paged_forward(desc, G, x[Op.Q], Kp, Vp, qo, after, table_after)
    for name in ("O", "L"):
        assert replayed[name].tobytes() == eager[name].tobytes(), name
    ref = reference({Op.Q: x[Op.Q], Op.K: x[Op.K], Op.V: x[Op.V], Op.dO: np.zeros_like(x[Op.Q])}, G, qo, ko_after, True)
    _check_reference(replayed, ref, qo, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_encode_rejects_invalid_paged_tables(mode):
    import torch
    desc = _descriptor(256, 128, 64, mode, 4, False)
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    t = torch.zeros(8, dtype=torch.int32, device="cuda")
    p = t.data_ptr()
    for c, paged, message in ((_constants(256, 128, 4, 2), mfa.PagedKV(0, 10, p, p, p, 4, 16), "count 0"),
                              (_constants(256, 128, 4, 2), mfa.PagedKV(2, 10, p, p, p, 4, 24), "page_size 24"),
                              (_constants(256, 128, 4, 2), mfa.PagedKV(2, 10, p, 0, p, 4, 16), "column_lengths"),
                              (_constants(256, 128, 4, 2), mfa.PagedKV(2, 10, p, p, p, 0, 16), "page_stride 0"),
                              (_constants(0, 128, 4, 2), mfa.PagedKV(2, 10, p, p, p, 4, 16), "at least 1")):
        with pytest.raises(mfa.MFAError) as e:
            kernel.encode(c, {}, paged=paged)
        assert e.value.status == -2 and message in e.value.message, e.value.message
