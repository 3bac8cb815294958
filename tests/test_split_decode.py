"""Split-KV decode (AttentionKernel.encode(..., split=SplitKV(...)) with sequences= or paged=): the key range of each
packed or paged query tile may be cut into up to 16 ranges, each handled by a CTA of its own that leaves a partial
output, and a second launch merges the partials.

The plan (splitPlan) reads only host values and follows the documented rule.  On the GPU a split call meets the packed
and paged suites' tolerances against the float64 reference; a plan of one split is the existing call bit for bit; a
paged split call equals the packed split call on the same keys laid out contiguously for the same num_splits; two runs
agree bit for bit; empty sequences, chunks without keys, stale partials in the workspace and NaN outside a sequence's
keys never reach an output; and a captured split decode replays as the cache grows."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import mfa_b200 as mfa
import oracle
from tests.test_paged_kv import (PagedRun, _check_reference, _check_sentinels, _download_L, _outputs, _upload,
                                 build_pool, run_packed_forward)
from tests.test_varlen import _constants, _descriptor, _inputs, _offsets, reference
from tests.test_window import band_reference, windowed

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
SMS = 132   # what the library assumes without a device


# ------------------------------------------------------------------------------------------------ CPU: the API
def test_split_structs_and_version():
    assert ctypes.sizeof(mfa.SplitKV) == 8 and ctypes.sizeof(mfa.SplitPlan) == 16
    assert {n: getattr(mfa.SplitKV, n).offset for n, _ in mfa.SplitKV._fields_} == {"num_splits": 0, "max_column": 4}
    assert {n: getattr(mfa.SplitPlan, n).offset for n, _ in mfa.SplitPlan._fields_} == {
        "splits": 0, "heads_per_tile": 4, "grid_size": 8, "launch_count": 12}
    assert "split-KV decode" in mfa.version() and " 0.5 " in mfa.version() and "paged K/V" in mfa.version()


def _paged(S=2, max_row=1, stride=4, page=16):
    return mfa.PagedKV(S, max_row, 16, 16, 16, stride, page)   # (device pointers are not dereferenced on the host)


def _expect_error(call, message):
    with pytest.raises(mfa.MFAError) as e:
        call()
    assert e.value.status == -2 and message in e.value.message, e.value.message


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_invalid_split_requests_are_rejected(mode):
    desc = _descriptor(256, 128, 64, mode, 4, False)
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    c = _constants(256, 128, 4, 2)
    table = mfa.SequenceTable(2, 10, 10, 16, 16)
    plan = lambda **kw: kernel.splitPlan(c, **kw)   # noqa: E731
    _expect_error(lambda: plan(sequences=table, split=mfa.SplitKV(17)), "num_splits 17")
    _expect_error(lambda: plan(paged=_paged(), split=mfa.SplitKV(1000)), "num_splits 1000")
    _expect_error(lambda: plan(sequences=table, split=None), "NULL split")
    _expect_error(lambda: plan(sequences=table, paged=_paged(), split=mfa.SplitKV()), "both")
    _expect_error(lambda: plan(split=mfa.SplitKV()), "neither")
    # the tables' own checks, unchanged
    _expect_error(lambda: plan(paged=_paged(S=0), split=mfa.SplitKV()), "count 0")
    _expect_error(lambda: plan(paged=_paged(page=24), split=mfa.SplitKV()), "page_size 24")
    _expect_error(lambda: plan(sequences=mfa.SequenceTable(2, 300, 10, 16, 16), split=mfa.SplitKV()), "max_row 300")
    # encode: the same checks before any device work, and split= without a table
    for kw in ({"sequences": table}, {"paged": _paged()}):
        _expect_error(lambda: kernel.encode(c, {}, split=mfa.SplitKV(17), **kw), "num_splits 17")
    _expect_error(lambda: kernel.encode(c, {}, split=mfa.SplitKV()), "needs sequences= or paged=")
    arr = (ctypes.c_void_p * mfa.MFA_BUFFER_COUNT)()
    for fn, t in ((mfa._lib.mfa_attention_kernel_encode_sequences_split, table),
                  (mfa._lib.mfa_attention_kernel_encode_paged_split, _paged())):
        _expect_error(lambda: mfa._check(fn(kernel._handle, ctypes.byref(c._c), ctypes.byref(t), None,
                                            ctypes.byref(arr), None)), "NULL split")
    # backward kernels: only the forward
    for t in (KT.backwardQuery, KT.backwardKeyValue):
        backward = mfa.AttentionKernel(desc.kernelDescriptor(t))
        for kw in ({"sequences": table}, {"paged": _paged()}):
            _expect_error(lambda: backward.splitPlan(c, split=mfa.SplitKV(), **kw), "only the forward")
            _expect_error(lambda: backward.encode(c, {}, split=mfa.SplitKV(), **kw), "only the forward")


def expected_plan(kernel, c, table, split, policy, window=None, staged=0):
    """The documented rule, from host values: (splits, heads_per_tile, grid_size, launch_count)."""
    par, trav, _ = kernel.blockDimensions
    H = c._c.batch_count
    max_row, S = table.max_row, table.count
    bound = split.max_column or (table.max_column if isinstance(table, mfa.SequenceTable)
                                 else table.page_stride * table.page_size)
    G = c._c.kv_group
    hpt = G if 2 <= G <= par and max_row < par else 1   # the query heads of a K/V head share a tile
    tiles = -(-max_row // (par // hpt))
    H //= hpt
    blocks = -(-bound // trav)
    if window is not None:
        blocks = min(blocks, (par + window[0] + window[1] + trav - 1) // trav + 1)
    min_blocks, max_splits = policy
    if split.num_splits:
        splits = split.num_splits
    elif tiles * H * S * 2 > SMS or min_blocks == 0:
        splits = 1
    else:
        splits = 1
        for s in range(2, min(SMS // (tiles * H * S), max_splits, 16) + 1):
            if blocks // s >= min_blocks:
                splits = s
    return splits, hpt, tiles * splits * H * S, staged + 1 + (splits > 1)


PLANS = [  # (mode, D, H, G, S, max_row, Cs bound (sequence table max_column, or page_stride * P), split request)
    ("bf16", 128, 32, 8, 1, 1, 32768, (0, 0)),       # decode, long context: 8 heads per tile, 4 CTAs -> 8 splits
    ("bf16", 128, 32, 8, 64, 1, 4096, (0, 0)),       # many sequences: no split
    ("bf16", 64, 4, 1, 1, 1, 4096, (0, 0)),          # 4 CTAs: the table row's maximum of 8
    ("bf16", 64, 8, 2, 2, 1, 300, (0, 0)),           # 3 key blocks with at least 2 per range: 1 split
    ("fp16", 128, 6, 6, 2, 1, 5000, (0, 0)),         # 40 blocks, not a multiple of the 8 splits
    ("bf16", 128, 16, 8, 1, 200, 2048, (0, 0)),      # max_row > 128: unpacked, two tiles per head
    ("bf16", 128, 16, 8, 1, 128, 2048, (0, 0)),      # max_row = 128: unpacked
    ("bf16", 128, 16, 8, 1, 127, 2048, (0, 0)),      # max_row = 127: 8 heads of 16 rows, 8 tiles per K/V head
    ("bf16", 128, 256, 128, 1, 1, 4096, (0, 0)),     # G = 128: one row of each of 128 heads per tile
    ("bf16", 128, 256, 256, 1, 1, 4096, (0, 0)),     # G = 256: more heads than tile rows, unpacked
    ("bf16", 256, 4, 2, 1, 1, 32768, (0, 0)),        # D = 256: the table row never splits
    ("bf16", 128, 4, 1, 1, 1, 32768, (0, 1024)),     # the hint bounds the keys
    ("bf16", 128, 64, 8, 8, 16, 4096, (3, 0)),       # forced
    ("bf16", 128, 4, 4, 1, 1, 40, (16, 0)),          # forced, more ranges than key blocks
    ("reference", 70, 4, 2, 1, 1, 4096, (0, 0)),     # staged operands (packed calls only)
]


@pytest.mark.parametrize("layout", ["sequences", "paged"])
@pytest.mark.parametrize("mode,D,H,G,S,max_row,bound,ask", PLANS)
def test_split_plan_follows_the_rule(layout, mode, D, H, G, S, max_row, bound, ask):
    if layout == "paged" and D % 8:
        pytest.skip("paged calls on the tensor cores need D % 8 == 0")
    desc = _descriptor(4096, 65536, D, mode, H, True)
    kd = desc.kernelDescriptor(KT.forward)
    kernel = mfa.AttentionKernel(kd)
    c = _constants(4096, 65536, H, G)
    table = (mfa.SequenceTable(S, max_row, bound, 16, 16) if layout == "sequences" else
             mfa.PagedKV(S, max_row, 16, 16, 16, bound // 16, 16))
    split = mfa.SplitKV(*ask)
    staged = 4 if D % 8 and layout == "sequences" else 0   # Q, K, V staged, O copied back
    want = expected_plan(kernel, c, table, split, kd.splitPolicy, staged=staged)
    got = kernel.splitPlan(c, split=split, **{layout: table})
    assert (got.splits, got.heads_per_tile, got.grid_size, got.launch_count) == want, (kd.splitPolicy, want)
    # one split, one head per tile: the existing call's grid and launches
    if (got.splits, got.heads_per_tile) == (1, 1):
        assert got.grid_size == kernel.gridSize(c, **{layout: table})
        assert got.launch_count == kernel.launchCount(c, **{layout: table})


def test_split_plan_examples():
    """A few plans spelled out: FlashAttention-style long-context decode splits, a policy of (0, x) does not."""
    desc = _descriptor(4096, 65536, 128, "bf16", 32, True)
    kd = desc.kernelDescriptor(KT.forward)
    assert kd.splitPolicy == (4, 8)
    c = _constants(4096, 65536, 32, 8)
    paged = mfa.PagedKV(1, 1, 16, 16, 16, 32768 // 256, 256)
    plan = mfa.AttentionKernel(kd).splitPlan(c, paged=paged, split=mfa.SplitKV())
    # 8 query heads per tile: 4 CTAs, so 8 ranges of 32 blocks
    assert (plan.splits, plan.heads_per_tile, plan.grid_size, plan.launch_count) == (8, 8, 32, 2)
    kd.splitPolicy = (0, 8)
    plan = mfa.AttentionKernel(kd).splitPlan(c, paged=paged, split=mfa.SplitKV())
    assert (plan.splits, plan.heads_per_tile, plan.grid_size, plan.launch_count) == (1, 8, 4, 1)
    plan = mfa.AttentionKernel(kd).splitPlan(c, paged=paged, split=mfa.SplitKV(5))
    assert (plan.splits, plan.grid_size, plan.launch_count) == (5, 20, 2)
    # 128 query rows or more: one head per tile
    paged = mfa.PagedKV(1, 128, 16, 16, 16, 32768 // 256, 256)
    plan = mfa.AttentionKernel(kd).splitPlan(c, paged=paged, split=mfa.SplitKV(1))
    assert (plan.splits, plan.heads_per_tile, plan.grid_size, plan.launch_count) == (1, 1, 32, 1)


@pytest.mark.parametrize("window", [(100, 0), (4095, 0), (-1, 0)])
def test_split_plan_of_a_windowed_kernel(window):
    """The key-block bound of a windowed kernel is the band width of one tile when that is narrower."""
    desc = _descriptor(4096, 65536, 128, "bf16", 4, True)
    kd = desc.kernelDescriptor(KT.forward)
    kernel = mfa.AttentionKernel(kd, window=window)
    c = _constants(4096, 65536, 4, 1)
    for layout, table in (("sequences", mfa.SequenceTable(1, 1, 32768, 16, 16)),
                          ("paged", mfa.PagedKV(1, 1, 16, 16, 16, 32768 // 16, 16))):
        # (an unbounded side resolves to row + column: the pool's 32768 keys of the paged call)
        w = (window[0] if window[0] >= 0 else 4096 + (65536 if layout == "sequences" else 32768), 0)
        want = expected_plan(kernel, c, table, mfa.SplitKV(), kd.splitPolicy, window=w)
        got = kernel.splitPlan(c, split=mfa.SplitKV(), **{layout: table})
        assert (got.splits, got.heads_per_tile, got.grid_size, got.launch_count) == want, (layout, want)
    if window == (100, 0):
        assert want[0] == 1   # two or three blocks of 128 keys: too few for ranges of 4


def test_simt_family_always_plans_one_split():
    desc = _descriptor(4096, 65536, 64, "fp32", 8, True)
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    c = _constants(4096, 65536, 8, 2)
    for layout, table in (("sequences", mfa.SequenceTable(1, 1, 32768, 16, 16)),
                          ("paged", mfa.PagedKV(1, 1, 16, 16, 16, 2048, 16))):
        for n in (0, 1, 16):
            got = kernel.splitPlan(c, split=mfa.SplitKV(n), **{layout: table})
            assert (got.splits, got.heads_per_tile) == (1, 1)
            assert got.grid_size == kernel.gridSize(c, **{layout: table})
            assert got.launch_count == kernel.launchCount(c, **{layout: table})


def test_cpp_host_mirror_with_split_kv(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  AttentionDescriptor d;
  d.lowPrecisionInputs = true;
  d.matrixDimensions = MatrixDimensions{300, 65536, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  d.batchCount = 32;
  d.causal = true;
  mfa_function_constants_t constants;
  d.setFunctionConstants(constants);
  kvGroup(constants) = 8;
  static int32_t fake[3];
  PagedKV paged{1, 1, fake, fake, fake, 128, 256};
  SequenceTable sequences{1, 1, 32768, fake, fake};
  AttentionKernel f(d.kernelDescriptor(AttentionKernelType::forward));
  const SplitPlan a = f.splitPlan(constants, paged, SplitKV{0, 0});
  const SplitPlan b = f.splitPlan(constants, sequences, SplitKV{3, 0});
  std::printf("%u %u %u %u %u %u %zu %zu\n", a.splits, a.heads_per_tile, a.grid_size, a.launch_count, b.splits,
              b.grid_size, sizeof(SplitKV), sizeof(SplitPlan));
  try {
    f.splitPlan(constants, paged, SplitKV{17, 0});
  } catch (const std::exception &e) {
    std::printf("rejected\n");
  }
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", root, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert out == ["8", "8", "32", "2", "3", "12", "8", "16", "rejected"], out


def test_ptxas_split_kernels_have_no_spills_and_no_stack_frame():
    from tests.test_forward_pipeline import _ptxas_report
    report, text = _ptxas_report()
    kernels = {name: r for name, r in report.items() if "split_forward_" in name}
    # 3 head-dimension chunk counts x bf16 / fp16 x (packed, paged) x (causal or not, or a window)
    assert len(kernels) == 3 * 2 * 2 * 3, sorted(kernels)
    merges = [name for name in report if "merge_sequence_splits" in name]
    assert len(merges) == 1, merges
    for name, r in list(kernels.items()) + [(merges[0], report[merges[0]])]:
        assert r == (0, 0, 0), (name, r)
        assert not re.search(r"C7510.*" + re.escape(name), text), name


# ------------------------------------------------------------------------------------------------ GPU
def run_packed_split(desc, G, Q, K, V, qo, ko, split, stream=0):
    """run_packed_forward through encode(..., sequences=, split=)."""
    import torch
    prec = desc.memoryPrecisions
    H, T, D = Q.shape
    q, k, v = _upload(Q, prec[Op.Q]), _upload(K, prec[Op.K]), _upload(V, prec[Op.V])
    O, L = _outputs(H, T, D, prec[Op.L])
    tq, tk = (torch.tensor(x, dtype=torch.int32, device="cuda") for x in (qo, ko))
    rq, rk = np.diff(qo), np.diff(ko)
    table = mfa.SequenceTable(len(qo) - 1, max(1, int(rq.max())), max(1, int(rk.max())), tq.data_ptr(), tk.data_ptr())
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
    kernel.encode(_constants(T, K.shape[1], H, G),
                  {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(), Op.L: L.data_ptr()},
                  stream, sequences=table, split=split)
    torch.cuda.synchronize()
    return {"O": O.cpu().numpy().reshape(H, T, D), "L": _download_L(L, prec[Op.L], H, T)}


class SplitPagedRun(PagedRun):
    def __init__(self, *args, split=None, **kw):
        super().__init__(*args, **kw)
        self.split = split

    def encode(self, stream=0):
        self.kernel.encode(self.constants, {Op.Q: self.q.data_ptr(), Op.K: self.k.data_ptr(), Op.V: self.v.data_ptr(),
                                            Op.O: self.O.data_ptr(), Op.L: self.L.data_ptr()},
                           stream, paged=self.paged, split=self.split)

    def plan(self):
        return self.kernel.splitPlan(self.constants, paged=self.paged, split=self.split)


def run_paged_split(desc, G, Q, Kp, Vp, qo, lengths, table, split):
    run = SplitPagedRun(desc, G, Q, Kp, Vp, qo, lengths, table, split=split)
    run.encode()
    return run.results()


def run_paged_plain(desc, G, Q, Kp, Vp, qo, lengths, table):
    run = PagedRun(desc, G, Q, Kp, Vp, qo, lengths, table)
    run.encode()
    return run.results()


def _same(a, b, rows=None):
    for name in ("O", "L"):
        x, y = (a[name], b[name]) if rows is None else (a[name][:, :rows], b[name][:, :rows])
        assert x.tobytes() == y.tobytes(), name


LENGTHS = {  # (query lengths Rs, key lengths Cs)
    "decode": ([1, 1, 1, 1, 1], [1, 40, 129, 1000, 3000]),
    "prefill": ([1, 100, 200, 5], [700, 300, 900, 5]),      # a chunked-prefill row and a two-tile sequence
    "empty": ([3, 0, 70, 1], [90, 50, 0, 600]),             # Rs = 0, Cs = 0
}
CASES = [  # (mode, D, causal, window, G, num_splits, page size, lengths)
    ("bf16", 128, True, None, 4, 0, 16, "decode"),
    ("bf16", 128, False, None, 1, 2, 256, "prefill"),
    ("bf16", 64, True, None, 8, 3, 16, "empty"),
    ("bf16", 256, True, None, 4, 16, 64, "decode"),
    ("fp16", 64, False, None, 4, 16, 256, "decode"),
    ("fp16", 128, True, (100, 0), 8, 3, 16, "prefill"),
    ("fp16", 256, False, None, 1, 2, 16, "empty"),
    ("reference", 128, True, None, 8, 2, 64, "decode"),
    ("reference", 64, False, (40, 20), 4, 3, 16, "prefill"),
    ("bf16", 64, True, (63, 0), 1, 16, 16, "decode"),
    ("bf16", 128, True, None, 4, 1, 16, "decode"),      # one split: the existing kernel
    ("fp16", 128, True, None, 1, 0, 256, "empty"),
]


def _case(mode, D, causal, G, lengths, page_size, seed):
    rq, rk = LENGTHS[lengths]
    qo, ko = _offsets(rq), _offsets(rk)
    H = 8
    T, Tk = qo[-1] + 9, ko[-1] + 5   # query rows past the table's end keep their sentinels
    desc = _descriptor(T, Tk, D, mode, H, causal)
    x = _inputs(desc, G, T, Tk, seed)
    Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, page_size, np.random.default_rng(seed))
    return desc, x, qo, ko, rk, Kp, Vp, table


def _reference(x, G, qo, ko, causal, window):
    inputs = {Op.Q: x[Op.Q], Op.K: x[Op.K], Op.V: x[Op.V], Op.dO: np.zeros_like(x[Op.Q])}
    if window is None:
        return reference(inputs, G, qo, ko, causal)
    return band_reference(inputs, G, qo, ko, window[0], 0 if causal else window[1])


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,window,G,num_splits,page_size,lengths", CASES)
def test_split_calls_meet_the_reference_and_the_existing_calls(mode, D, causal, window, G, num_splits, page_size,
                                                               lengths):
    """Paged and packed split calls against the float64 reference; paged = packed bitwise for the same num_splits; two
    runs agree bitwise; a plan of one split is the existing call bitwise."""
    import contextlib
    desc, x, qo, ko, rk, Kp, Vp, table = _case(mode, D, causal, G, lengths, page_size, seed=D + G + page_size)
    split = mfa.SplitKV(num_splits)
    with (windowed(window) if window else contextlib.nullcontext()):
        run = SplitPagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, split=split)
        plan = run.plan()
        run.encode()
        paged = run.results()
        run.O.fill_(float("nan"))
        run.L.fill_(float("nan"))
        run.encode()
        again = run.results()
        packed = run_packed_split(desc, G, x[Op.Q], x[Op.K], x[Op.V], qo, ko, split)
        if num_splits == 1:
            # one split, with or without the group's query heads in one tile: the existing calls bit for bit (a row's
            # arithmetic does not depend on the tile's other rows; blocks wholly masked for a row are exact no-ops)
            _same(paged, run_paged_plain(desc, G, x[Op.Q], Kp, Vp, qo, rk, table))
            _same(packed, run_packed_forward(desc, G, x[Op.Q], x[Op.K], x[Op.V], qo, ko))
    if num_splits:
        assert plan.splits == num_splits
    assert plan.heads_per_tile == (G if G > 1 and max(LENGTHS[lengths][0]) < 128 else 1)
    _same(paged, again)
    _check_sentinels(paged, qo)
    _check_sentinels(packed, qo)
    if num_splits:   # (the default plans of the two tables differ: their key bounds differ)
        _same(paged, packed, rows=qo[-1])
    ref = _reference(x, G, qo, ko, causal, window)
    _check_reference(paged, ref, qo, "fp16" if mode == "reference" else mode)
    _check_reference(packed, ref, qo, "fp16" if mode == "reference" else mode)


@pytest.mark.gpu
def test_packed_split_with_staged_operands():
    """D = 36: Q, K and V are staged with 40 columns and O copied back, around the split kernel and its merge."""
    desc, x, qo, ko, rk, _, _, _ = _case("bf16", 36, True, 2, "prefill", 16, seed=36)
    for n in (0, 3):
        out = run_packed_split(desc, 2, x[Op.Q], x[Op.K], x[Op.V], qo, ko, mfa.SplitKV(n))
        _check_sentinels(out, qo)
        _check_reference(out, reference({**x, Op.dO: np.zeros_like(x[Op.Q])}, 2, qo, ko, True), qo, "bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "reference"])
def test_stale_partials_and_nan_outside_the_keys_never_reach_an_output(mode):
    """A large split call on the stream first leaves finite partials in the workspace; then 16 splits over sequences of
    40 keys or none (chunks without keys), with NaN in every pool row past Cs and in spare pages, and page-table entries
    past the last page of -1 or a huge id: the outputs equal those of a clean pool bit for bit and meet the reference."""
    big_desc, bx, bqo, bko, brk, bKp, bVp, btable = _case(mode, 128, False, 4, "prefill", 64, seed=5)
    run_paged_split(big_desc, 4, bx[Op.Q], bKp, bVp, bqo, brk, btable, mfa.SplitKV(16))
    rq, rk = [1, 2, 1, 0], [40, 0, 40, 40]
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 9, ko[-1] + 5
    desc = _descriptor(T, Tk, 128, mode, 8, True)
    x = _inputs(desc, 4, T, Tk, seed=6)
    Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, 16, np.random.default_rng(6))
    clean = run_paged_split(desc, 4, x[Op.Q], Kp, Vp, qo, rk, table, mfa.SplitKV(16))
    for fill, tail in ((np.nan, -1), (np.inf, 2**31 - 1)):
        Kd, Vd, td = build_pool(x[Op.K], x[Op.V], ko, 16, np.random.default_rng(6), fill=fill, tail=tail)
        dirty = run_paged_split(desc, 4, x[Op.Q], Kd, Vd, qo, rk, td, mfa.SplitKV(16))
        _check_sentinels(dirty, qo)
        _same(clean, dirty)
    _check_reference(clean, reference({**x, Op.dO: np.zeros_like(x[Op.Q])}, 4, qo, ko, True), qo,
                     "fp16" if mode == "reference" else mode)


@pytest.mark.gpu
def test_windowed_split_never_reads_pages_outside_the_band():
    """A (63, 0) window over 3000 keys in 8 ranges: pages wholly before the band point at a NaN page or far outside the
    pool, and the output is bitwise that of the clean table."""
    rq, rk = [1, 1], [3000, 700]
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 9, ko[-1] + 5
    desc = _descriptor(T, Tk, 64, "bf16", 4, True)
    x = _inputs(desc, 2, T, Tk, seed=8)
    Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, 16, np.random.default_rng(8))
    with windowed((63, 0)):
        clean = run_paged_split(desc, 2, x[Op.Q], Kp, Vp, qo, rk, table, mfa.SplitKV(8))
        Kn, Vn = (np.concatenate([p_, np.full((1,) + p_.shape[1:], np.nan, np.float32)]) for p_ in (Kp, Vp))
        poisoned = table.copy()
        for s, Cs in enumerate(rk):
            first = (Cs - 1 - 63) // 16   # pages wholly before the band of the one query row
            poisoned[s, :first] = [Kn.shape[0] - 1 if j % 2 else 2**31 - 1 for j in range(first)]
        skipped = run_paged_split(desc, 2, x[Op.Q], Kn, Vn, qo, rk, poisoned, mfa.SplitKV(8))
    _same(clean, skipped)
    ref = band_reference({**x, Op.dO: np.zeros_like(x[Op.Q])}, 2, qo, ko, 63, 0)
    _check_reference(clean, ref, qo, "bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_split_decode_replays_in_a_cuda_graph_as_the_cache_grows(mode):
    """A captured split decode step (library plan: one sequence, long context) replayed after column_lengths and
    page_table grew by a token equals a fresh call bit for bit, and the reference."""
    import torch
    page_size, G, H, D = 16, 4, 8, 128
    before = [2047, 15]
    after = [c + 1 for c in before]
    qo = _offsets([1] * len(before))
    T = qo[-1]
    desc = _descriptor(T, 4096, D, mode, H, True)
    prec = desc.memoryPrecisions
    rng = np.random.default_rng(31)
    x = {op: oracle.roundtrip(rng.standard_normal(shape).astype(np.float32), int(prec[op]))
         for op, shape in ((Op.Q, (H, T, D)), (Op.K, (H // G, sum(after), D)), (Op.V, (H // G, sum(after), D)))}
    ko_after = _offsets(after)
    Kp, Vp, table_after = build_pool(x[Op.K], x[Op.V], ko_after, page_size, rng, spare_pages=8)
    table_before = table_after.copy()
    for s, c in enumerate(before):
        table_before[s, -(-c // page_size):] = -1
    run = SplitPagedRun(desc, G, x[Op.Q], Kp, Vp, qo, before, table_before, split=mfa.SplitKV())
    if mode == "bf16":
        assert run.plan().splits > 1
    stream = torch.cuda.Stream()
    run.encode(stream.cuda_stream)   # (outside any capture first, on the capturing stream: its workspace)
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        run.encode(stream.cuda_stream)
    run.lengths.copy_(torch.tensor(after, dtype=torch.int32))
    run.table.copy_(torch.tensor(table_after, dtype=torch.int32))
    run.O.fill_(float("nan"))
    run.L.fill_(float("nan"))
    graph.replay()
    replayed = run.results()
    fresh = run_paged_split(desc, G, x[Op.Q], Kp, Vp, qo, after, table_after, mfa.SplitKV())
    _same(replayed, fresh)
    ref = reference({Op.Q: x[Op.Q], Op.K: x[Op.K], Op.V: x[Op.V], Op.dO: np.zeros_like(x[Op.Q])}, G, qo, ko_after, True)
    _check_reference(replayed, ref, qo, mode)


@pytest.mark.gpu
def test_simt_split_calls_equal_the_existing_calls():
    desc, x, qo, ko, rk, Kp, Vp, table = _case("fp32", 72, True, 4, "prefill", 16, seed=9)
    for n in (0, 4):
        _same(run_paged_split(desc, 4, x[Op.Q], Kp, Vp, qo, rk, table, mfa.SplitKV(n)),
              run_paged_plain(desc, 4, x[Op.Q], Kp, Vp, qo, rk, table))
        _same(run_packed_split(desc, 4, x[Op.Q], x[Op.K], x[Op.V], qo, ko, mfa.SplitKV(n)),
              run_packed_forward(desc, 4, x[Op.Q], x[Op.K], x[Op.V], qo, ko))


@pytest.mark.gpu
def test_plan_counts_match_a_profiler_trace():
    """launch_count and grid_size of splitPlan against the kernels a torch.profiler trace of one encode records."""
    import json
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = f"import json, sys; sys.path.insert(0, {root!r}); from tests.test_split_decode import _trace_launches; " \
           f"print(json.dumps(_trace_launches()))"
    proc = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-4000:]
    results = json.loads(proc.stdout.strip().splitlines()[-1])
    for name, (launched, grids, plan) in results.items():
        assert len(launched) == plan[3], (name, launched, plan)
        assert grids[0] == plan[2], (name, grids, plan)   # the attention kernel goes first (after any staging)
    assert results["bf16 D=128 paged n=0"][2][0] > 1 and results["bf16 D=36 packed n=3"][2][3] == 4 + 2


def _trace_launches():
    """{case: (library kernels in a torch.profiler trace of one encode, their grid sizes without staging, the plan)},
    run in a process of its own (the profiler's state is process-wide)."""
    import json
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for mode, D, layout, n in (("bf16", 128, "paged", 0), ("bf16", 128, "packed", 1), ("bf16", 36, "packed", 3),
                               ("fp16", 64, "paged", 16)):
        desc, x, qo, ko, rk, Kp, Vp, table = _case(mode, D, True, 4, "decode", 16, seed=D)
        split = mfa.SplitKV(n)
        if layout == "paged":
            run = SplitPagedRun(desc, 4, x[Op.Q], Kp, Vp, qo, rk, table, split=split)
            plan, encode = run.plan(), run.encode
        else:
            prec = desc.memoryPrecisions
            H, T, _ = x[Op.Q].shape
            q, k, v = _upload(x[Op.Q], prec[Op.Q]), _upload(x[Op.K], prec[Op.K]), _upload(x[Op.V], prec[Op.V])
            O, L = _outputs(H, T, D, prec[Op.L])
            tq, tk = (torch.tensor(a, dtype=torch.int32, device="cuda") for a in (qo, ko))
            seq = mfa.SequenceTable(len(qo) - 1, 1, int(np.diff(ko).max()), tq.data_ptr(), tk.data_ptr())
            kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
            c = _constants(T, x[Op.K].shape[1], H, 4)
            ptrs = {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(), Op.L: L.data_ptr()}
            plan = kernel.splitPlan(c, sequences=seq, split=split)
            encode = lambda: kernel.encode(c, ptrs, sequences=seq, split=split)   # noqa: E731
        encode()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            torch.zeros(1, device="cuda").add_(0.0)   # (the trace can miss the first kernel of the window)
            torch.cuda.synchronize()
            encode()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as tmp:
            prof.export_chrome_trace(os.path.join(tmp, "trace.json"))
            with open(os.path.join(tmp, "trace.json")) as f:
                trace = json.load(f)
        kernels = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel" and "mfa::" in e.get("name", "")),
                         key=lambda e: e["ts"])
        launched = [e["name"] for e in kernels]
        grids = [int(np.prod(e["args"]["grid"])) for e in kernels if "stage" not in e["name"]]
        out[f"{mode} D={D} {layout} n={n}"] = (launched, grids, [plan.splits, plan.heads_per_tile, plan.grid_size,
                                                                 plan.launch_count])
    return out
