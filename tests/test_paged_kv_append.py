"""Paged K/V append (appendPagedKV(paged, PagedKVAppend(...), k_pool, v_pool, fp8=)): a step's new keys and values,
packed by sequence as the paged forward's queries, are written into the page pools through the forward's own table.

New token i of sequence s (0 <= i < Rs) becomes key p = Cs - Rs + i, pool row page_table[s][p // P] * P + p % P, every
K/V head.  The reference below computes that slot mapping from the same tables, with the forward's clamping (query
ranges into [0, rows], Cs into [0, page_stride * P]) and the append's skipping (p < 0, or a page id outside [0, pages)).
On the GPU the written rows must equal it byte for byte, and every other byte of both pools, a guard tail past
pool_rows included, must keep its sentinel.  FP8 pools hold (x.float() / scale).clamp(-448, 448).to(float8_e4m3fn),
with NaN checked as NaN.  An append followed by a paged forward equals the forward over pools filled by the torch
recipe bit for bit, and a captured decode step (append, then the split forward) replays as the cache grows."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import mfa_b200 as mfa

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3_MAX = 448.0


# ------------------------------------------------------------------------------------------------ the reference
def slot_mapping(row_offsets, lengths, table, page_size, rows, pool_rows):
    """[(source token, pool row)] of every write the append makes, from the tables as the kernel reads them"""
    stride = table.shape[1]
    pages = pool_rows // page_size
    out = []
    for s in range(len(lengths)):
        lo = min(max(int(row_offsets[s]), 0), rows)
        hi = min(max(int(row_offsets[s + 1]), lo), rows)
        Rs, Cs = hi - lo, min(max(int(lengths[s]), 0), stride * page_size)
        for i in range(Rs):
            p = Cs - Rs + i
            if p < 0:
                continue
            page = int(table[s, p // page_size])
            if 0 <= page < pages:
                out.append((lo + i, page * page_size + p % page_size))
    return out


def torch_slot_mapping(row_offsets, lengths, table, page_size):
    """The slot mapping of the recipe the append replaces, for well-formed tables: the new tokens of sequence s go to
    keys [Cs - Rs, Cs), looked up in its page_table row"""
    import torch
    new = np.diff(row_offsets)
    keys = torch.cat([torch.arange(c - n, c) for c, n in zip(np.asarray(lengths).tolist(), new.tolist())])
    seq = torch.cat([torch.full((n,), s) for s, n in enumerate(new.tolist())])
    tbl = torch.as_tensor(table)
    return (tbl[seq, keys // page_size] * page_size + keys % page_size).tolist()


def e4m3_reference(x, scales):
    """torch's saturating recipe: x [T][Hkv][D] (any float dtype) / per-head scales -> E4M3 bytes, uint8 [T][Hkv][D]"""
    import torch
    s = torch.ones(x.shape[1]) if scales is None else torch.as_tensor(np.asarray(scales, np.float32))
    q = (x.float() / s[None, :, None]).clamp(-E4M3_MAX, E4M3_MAX)
    return q.to(torch.float8_e4m3fn).view(torch.uint8)


# ------------------------------------------------------------------------------------------------ CPU: the API
def test_append_struct_and_version():
    assert ctypes.sizeof(mfa.PagedKVAppend) == 40
    offsets = {name: getattr(mfa.PagedKVAppend, name).offset for name, _ in mfa.PagedKVAppend._fields_}
    assert offsets == {"k_new": 0, "v_new": 8, "rows": 16, "token_stride": 20, "kv_heads": 24, "head_dimension": 28,
                       "pool_rows": 32, "precision": 36}
    assert hasattr(mfa._lib, "mfa_paged_kv_append")
    assert "paged K/V append" in mfa.version() and " 0.5 " in mfa.version()
    assert "PagedKVAppend" in mfa.__all__ and "appendPagedKV" in mfa.__all__


def test_reference_slot_mapping_is_the_torch_recipe():
    """On well-formed tables the reference writes exactly the slots of the recipe it replaces, in token order."""
    rng = np.random.default_rng(0)
    rq, rk, P = [1, 0, 37, 1, 5], [1, 9, 100, 64, 5], 16
    qo = [0] + list(np.cumsum(rq))
    table = rng.permutation(64).reshape(8, 8)[:len(rq)]
    got = slot_mapping(qo, rk, table, P, qo[-1], 64 * P)
    assert [t for t, _ in got] == list(range(qo[-1]))
    assert [r for _, r in got] == torch_slot_mapping(qo, rk, table, P)


def _paged(S=2, max_row=4, rows=16, lengths=16, table=16, stride=4, page=16):
    return mfa.PagedKV(S, max_row, rows, lengths, table, stride, page)   # (device pointers are not dereferenced)


def _append(k=16, v=16, rows=8, stride=0, heads=2, D=64, pool_rows=256, prec=P.BF16):
    return mfa.PagedKVAppend(k, v, rows, stride, heads, D, pool_rows, prec)


def _expect_error(call, message):
    with pytest.raises(mfa.MFAError) as e:
        call()
    assert e.value.status == -2 and message in e.value.message, e.value.message


def test_invalid_appends_are_rejected():
    """Each rejection names its field, before any device work (no GPU is needed to reach them)."""
    bad = [(None, _append(), "NULL paged K/V table"),
           (_paged(), None, "NULL append"),
           (_paged(), _append(k=0), "k_new must not be NULL"),
           (_paged(), _append(v=0), "v_new must not be NULL"),
           (_paged(rows=0), _append(), "row_offsets must not be NULL"),
           (_paged(lengths=0), _append(), "column_lengths must not be NULL"),
           (_paged(table=0), _append(), "page_table must not be NULL"),
           (_paged(S=0), _append(), "count 0 is outside [1, 65535]"),
           (_paged(S=65536), _append(), "count 65536 is outside [1, 65535]"),
           (_paged(max_row=0), _append(), "max_row 0 is outside [1, rows = 8]"),
           (_paged(max_row=9), _append(), "max_row 9 is outside [1, rows = 8]"),
           (_paged(page=24), _append(), "page_size 24 must be a power of two, at least 16, dividing pool_rows = 256"),
           (_paged(page=8), _append(), "page_size 8"),
           (_paged(page=512), _append(), "page_size 512"),
           (_paged(stride=0), _append(), "page_stride 0 must be at least 1"),
           (_paged(), _append(heads=0), "kv_heads 0 must be at least 1"),
           (_paged(), _append(D=0), "head_dimension 0 is outside [1, 512]"),
           (_paged(), _append(D=513), "head_dimension 513 is outside [1, 512]"),
           (_paged(), _append(stride=127), "token_stride 127 is below kv_heads * head_dimension = 128"),
           (_paged(), _append(prec=3), "precision 3 is not MFA_FP32, MFA_FP16 or MFA_BF16")]
    for paged, append, message in bad:
        _expect_error(lambda: mfa.appendPagedKV(paged, append, 16, 16), message)
        _expect_error(lambda: mfa.appendPagedKV(paged, append, 16, 16, fp8=mfa.FP8KV()), message)
    _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(), 0, 16), "k_pool must not be NULL")
    _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(), 16, 0), "v_pool must not be NULL")


def test_forward_table_messages_are_unchanged():
    """The forward's table checks, now shared with the append, keep their wording (row / column, not the append's)."""
    from tests.test_varlen import _constants, _descriptor
    kernel = mfa.AttentionKernel(_descriptor(256, 128, 64, "bf16", 4, False).kernelDescriptor(KT.forward))
    c = _constants(256, 128, 4, 2)
    _expect_error(lambda: kernel.encode(c, {}, paged=_paged(max_row=300)), "max_row 300 is outside [1, row = 256].")
    _expect_error(lambda: kernel.encode(c, {}, paged=_paged(page=24)),
                  "page_size 24 must be a power of two, at least 16, dividing column = 128.")


def test_cpp_host_mirror_of_the_append(tmp_path):
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include <cstring>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  static int32_t fake[4];
  const PagedKV paged{1, 1, fake, fake, fake, 4, 16};
  const PagedKVAppend append{fake, fake, 1, 0, 0, 64, 64, MFA_BF16};   // kv_heads 0
  const FP8KV fp8{nullptr, nullptr};
  for (const FP8KV *f : {static_cast<const FP8KV *>(nullptr), &fp8}) {
    try {
      appendPagedKV(paged, append, fake, fake, f);
    } catch (const std::exception &e) {
      std::printf("%s\n", std::strstr(e.what(), "kv_heads 0") ? "rejected" : e.what());
    }
  }
  std::printf("%zu\n", sizeof(PagedKVAppend));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    assert out[:3] == ["rejected", "rejected", "40"], out


def test_ptxas_append_kernels_have_no_spills_and_no_stack_frame():
    log = os.path.join(ROOT, "metal-flash-attention_b200", "_build", "kernels", "paged_append.o.ptxas.log")
    assert os.path.exists(log), f"{log} is missing: build() writes it when it compiles the library"
    text = open(log).read()
    report, function = {}, None
    for line in text.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            function = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and function is not None:
            report[function] = tuple(int(x) for x in m.groups())
            function = None
    kernels = {name: r for name, r in report.items() if "paged_kv_append" in name}
    # FP32 / FP16 / BF16 sources x (copy, E4M3) x (vector, scalar)
    assert len(kernels) == 12, sorted(kernels)
    assert all(r == (0, 0, 0) for r in kernels.values()), kernels


# ------------------------------------------------------------------------------------------------ GPU
# Each GPU check runs in a process of its own, as the FP8 K/V suite's do: the launch-count tests of other suites record
# torch.profiler traces that are fragile to what ran before them in the same process.
def _isolated(check, *args):
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_paged_kv_append as t; "
            f"t.{check}(*{args!r})")
    proc = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]


TORCH_DTYPE = {"fp32": "float32", "fp16": "float16", "bf16": "bfloat16"}
PREC = {"fp32": P.FP32, "fp16": P.FP16, "bf16": P.BF16}
LENGTHS = {  # (new tokens Rs, cache lengths Cs with them)
    # decode, a chunk crossing pages with Cs - Rs not page-aligned, Rs = 0, a chunk starting at key 0, and a mix
    "mixed": ([1, 40, 0, 1, 300, 17], [1, 75, 33, 258, 300, 17 + 5]),
    "decode": ([1] * 7, [1, 2, 16, 17, 64, 257, 1000]),
}


class AppendCase:
    """Device buffers of one append: sources k_new / v_new [rows][Hkv][D] (or slices of a fused
    [rows][H + 2 Hkv][D] projection), tables, and pools of pool_rows rows plus a guard tail, filled with random
    sentinel bytes.  Source rows outside every sequence hold NaN."""

    def __init__(self, dtype, page_size, Hkv, D, rq, rk, seed, fused=False, fp8=None, table=None, row_offsets=None,
                 pages=None, extra_pages=4, guard_rows=7, values=None):
        import torch
        self.torch = torch
        rng = np.random.default_rng(seed)
        self.P, self.Hkv, self.D = page_size, Hkv, D
        qo = row_offsets if row_offsets is not None else [2] + list(2 + np.cumsum(rq))
        self.qo = np.asarray(qo, np.int64)
        self.rows = int(max(self.qo.max(), 0)) + 3   # (rows before the first and after the last sequence)
        if table is None:
            pages_of = [-(-max(int(c), 0) // page_size) for c in rk]
            stride = max(1, max(pages_of))
            num_pages = sum(pages_of) + extra_pages
            order = rng.permutation(num_pages)
            table = np.full((len(rk), stride), -1, np.int64)
            n = 0
            for s, count in enumerate(pages_of):
                table[s, :count] = order[n:n + count]
                n += count
            self.pool_rows = num_pages * page_size
        else:
            self.pool_rows = (pages or int(np.asarray(table).max()) + 1 + extra_pages) * page_size
        self.table_np = np.asarray(table, np.int64)
        self.lengths_np = np.asarray(rk, np.int64)
        dt = getattr(torch, TORCH_DTYPE[dtype])
        self.prec = PREC[dtype]
        H = 3
        if values is None:
            values = torch.from_numpy(rng.standard_normal((self.rows, H + 2 * Hkv, D)).astype(np.float32)) * 2
        else:
            values = values.reshape(self.rows, H + 2 * Hkv, D)
        fused_t = values.to(dt)
        inside = np.zeros(self.rows, bool)
        for s in range(len(rk)):
            lo = min(max(int(self.qo[s]), 0), self.rows)
            inside[lo:min(max(int(self.qo[s + 1]), lo), self.rows)] = True
        fused_t[torch.from_numpy(~inside)] = float("nan")
        self.fused = fused_t.cuda()
        if fused:
            self.k_new, self.v_new = self.fused[:, H:H + Hkv], self.fused[:, H + Hkv:]
            self.token_stride = (H + 2 * Hkv) * D
        else:
            self.k_new = self.fused[:, H:H + Hkv].contiguous()
            self.v_new = self.fused[:, H + Hkv:].contiguous()
            self.token_stride = 0
        self.fp8 = fp8
        self.row_bytes = Hkv * D * (1 if fp8 is not None else fused_t.element_size())
        total = (self.pool_rows + guard_rows) * self.row_bytes
        g = torch.Generator(device="cuda")
        g.manual_seed(seed)
        self.k_pool, self.v_pool = (torch.randint(0, 256, (total,), dtype=torch.uint8, device="cuda", generator=g)
                                    for _ in range(2))
        self.k_before, self.v_before = self.k_pool.clone(), self.v_pool.clone()
        self.row_offsets = torch.tensor(self.qo, dtype=torch.int32, device="cuda")
        self.lengths = torch.tensor(np.clip(self.lengths_np, -2**31, 2**31 - 1), dtype=torch.int32, device="cuda")
        self.table = torch.tensor(np.clip(self.table_np, -2**31, 2**31 - 1), dtype=torch.int32, device="cuda")
        max_row = max(1, int(np.max(np.diff(np.clip(self.qo, 0, self.rows)), initial=1)))
        self.paged = mfa.PagedKV(len(rk), max_row, self.row_offsets.data_ptr(), self.lengths.data_ptr(),
                                 self.table.data_ptr(), self.table_np.shape[1], page_size)
        self.scales = None
        self.fp8_arg = None
        if fp8 is not None:
            self.scales = [None if s is None else torch.tensor(np.asarray(s, np.float32), device="cuda") for s in fp8]
            self.fp8_arg = mfa.FP8KV(*(0 if s is None else s.data_ptr() for s in self.scales))

    def append(self, stream=0):
        a = mfa.PagedKVAppend(self.k_new.data_ptr(), self.v_new.data_ptr(), self.rows, self.token_stride, self.Hkv,
                              self.D, self.pool_rows, self.prec)
        mfa.appendPagedKV(self.paged, a, self.k_pool.data_ptr(), self.v_pool.data_ptr(), fp8=self.fp8_arg,
                          stream=stream)

    def check(self):
        """Written rows equal the reference byte for byte (NaN as NaN in FP8 pools); every other byte is unchanged"""
        torch = self.torch
        torch.cuda.synchronize()
        slots = slot_mapping(self.qo, self.lengths_np, self.table_np, self.P, self.rows, self.pool_rows)
        for src, after, before, which in ((self.k_new, self.k_pool, self.k_before, 0),
                                          (self.v_new, self.v_pool, self.v_before, 1)):
            expected = before.clone().view(-1, self.row_bytes)
            got = after.view(-1, self.row_bytes)
            if slots:
                tokens = torch.tensor([t for t, _ in slots], device="cuda")
                rows = torch.tensor([r for _, r in slots], device="cuda")
                x = src[tokens].cpu()
                if self.fp8 is None:
                    want = x.contiguous().view(torch.uint8).reshape(len(slots), self.row_bytes)
                else:
                    want = e4m3_reference(x, self.fp8[which]).reshape(len(slots), self.row_bytes)
                    nan = (want & 0x7F) == 0x7F
                    have = got[rows].cpu()
                    assert ((have[nan] & 0x7F) == 0x7F).all(), "NaN stays NaN"
                    want = torch.where(nan, have, want)
                expected[rows] = want.cuda()
            diff = (expected != got).any(dim=1).nonzero().flatten().tolist()
            assert not diff, f"{'KV'[which]} pool rows differ from the reference: {diff[:10]} (pool_rows " \
                             f"{self.pool_rows}, {len(slots)} written)"
        return slots


COPY_CASES = [  # (dtype, P, Hkv, D, fused)
    ("bf16", 16, 8, 128, False), ("fp16", 64, 2, 64, False), ("bf16", 256, 1, 256, True),
    ("fp16", 16, 8, 256, True), ("bf16", 64, 2, 128, False), ("fp16", 256, 1, 64, False),
    ("bf16", 64, 1, 36, False), ("fp16", 16, 2, 36, True),          # rows or strides not 16-byte multiples: scalar
    ("fp32", 64, 2, 40, False), ("fp32", 16, 1, 72, True), ("fp32", 256, 2, 33, False), ("fp32", 16, 8, 128, False),
]


@pytest.mark.gpu
def test_copy_appends_write_exactly_the_reference_rows():
    """16-bit and FP32 pools, P 16/64/256, Hkv 1/2/8, D 33..256, contiguous and fused sources, decode and mixed
    tables: the named rows hold the source's bits, every other byte (guard tail included) its sentinel."""
    _isolated("_check_cases", COPY_CASES, False)


FP8_CASES = [  # (dtype, P, Hkv, D, fused, scaled)
    ("bf16", 16, 8, 128, False, True), ("fp16", 64, 2, 64, True, True), ("fp32", 256, 1, 128, False, True),
    ("bf16", 64, 2, 40, False, False), ("fp16", 16, 1, 72, False, True), ("fp32", 16, 2, 36, True, True),
    ("bf16", 256, 8, 256, True, False), ("fp32", 64, 1, 40, False, False), ("fp16", 256, 2, 128, False, False),
]


@pytest.mark.gpu
def test_fp8_appends_write_the_saturating_torch_bytes():
    """E4M3 pools: bytes equal (x.float() / scale).clamp(-448, 448).to(float8_e4m3fn) for arbitrary per-head scales
    and NULL scales, over values past 448, +-inf, NaN, ties and subnormal results."""
    _isolated("_check_cases", FP8_CASES, True)


def _special_values(rng, n, dtype):
    """Random values with every special the conversion must get right: past 448, +-inf, NaN, ties to even in E4M3
    (at scale 1), subnormal E4M3 results, zeros"""
    import torch
    v = rng.standard_normal(n).astype(np.float32) * 30
    specials = np.array([448, 449, 463, 464, 500, 1e6, np.inf, -np.inf, np.nan, -0.0, 0.0, 1.0625, 1.1875, -1.0625,
                         3 * 2.0 ** -10, 2.0 ** -10, 5 * 2.0 ** -11, 2.0 ** -12, 240.0, 232.0, -464, 1e-3, 6e-3],
                        np.float32)
    idx = rng.choice(n, size=n // 8, replace=False)
    v[idx] = specials[rng.integers(0, len(specials), len(idx))]
    small = rng.choice(n, size=n // 8, replace=False)
    v[small] = rng.standard_normal(len(small)).astype(np.float32) * 2.0 ** -8
    return torch.from_numpy(v)


def _check_cases(cases, fp8):
    for n, case in enumerate(cases):
        dtype, P_, Hkv, D, fused = case[:5]
        for lengths in ("mixed", "decode"):
            rq, rk = LENGTHS[lengths]
            seed = 100 * n + len(lengths)
            scales = None
            values = None
            if fp8:
                rng = np.random.default_rng(seed)
                rows = 2 + sum(rq) + 3
                values = _special_values(rng, rows * (3 + 2 * Hkv) * D, dtype)
                if case[5]:
                    scales = tuple((rng.uniform(0.05, 3.0, Hkv) * (1 + 1 / 3)).astype(np.float32) for _ in range(2))
                else:
                    scales = (None, None)
            c = AppendCase(dtype, P_, Hkv, D, rq, rk, seed, fused=fused, fp8=scales, values=values)
            c.append()
            slots = c.check()
            assert len(slots) == sum(rq), (case, lengths)


@pytest.mark.gpu
def test_malformed_tables_write_nothing_they_should_not():
    """Rs > Cs, Cs past page_stride * P, negative Cs, page ids -1 and pool_rows / P, decreasing row offsets and rows
    outside every sequence (NaN): only the rows the reference names are written, and no NaN reaches a pool."""
    _isolated("_check_malformed")


def _check_malformed():
    P_ = 16
    rk = [2, 10_000, 40, 40, 40, -5, 30, 5]
    row_offsets = [2, 7, 10, 13, 16, 19, 21, 18, 22]   # (sequence 6 ends below its start: empty)
    table = np.array([[0, 1, 2],            # Rs = 5 > Cs = 2: only keys 0 and 1
                      [3, -1, 4],           # Cs clamped to 48: keys 45..47 on page 4
                      [5, 6, -1],           # keys 37..39 on page -1: skipped
                      [7, 8, 21],           # keys 37..39 on page 21 = pool_rows / P: skipped
                      [9, 10, 2**31 - 1],   # keys 37..39 on page 2^31 - 1: skipped
                      [11, 12, 13],         # Cs < 0 counts as 0: every p < 0
                      [14, 15, 15],
                      [16, 20, 20]], np.int64)   # Rs = 4 of Cs = 5: keys 1..4
    for dtype, fp8 in (("bf16", None), ("fp32", (np.array([0.37], np.float32), None))):
        c = AppendCase(dtype, P_, 1, 64, None, rk, 7, table=table, row_offsets=row_offsets, pages=21, fp8=fp8)
        assert c.pool_rows == 21 * P_
        c.append()
        slots = c.check()
        written = sorted(r for _, r in slots)
        assert written == [0, 1, 4 * P_ + 13, 4 * P_ + 14, 4 * P_ + 15] + [16 * P_ + i for i in range(1, 5)], written


@pytest.mark.gpu
def test_pages_past_two_gigabytes():
    """A page whose bytes start past 2^31 in an FP8 pool and in a 16-bit pool: 64-bit offsets."""
    _isolated("_check_far_pages")


def _check_far_pages():
    import torch
    P_, Hkv, D = 64, 8, 128
    for dtype, fp8, row_bytes in (("bf16", None, 2 * Hkv * D), ("bf16", (None, None), Hkv * D)):
        far = 2**31 // (row_bytes * P_)          # the first page whose bytes start at or past 2^31
        table = np.array([[0, far + 1], [far, 3]], np.int64)
        c = AppendCase(dtype, P_, Hkv, D, [3, 70], [P_ + 3, 70], 11, table=table, extra_pages=2, guard_rows=1, fp8=fp8)
        assert (far + 1) * P_ * c.row_bytes > 2**31 and far * P_ * c.row_bytes >= 2**31
        c.append()
        slots = c.check()
        assert {r // P_ for _, r in slots} == {far + 1, far, 3}
        del c
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ GPU: end to end
E2E = [  # (mode, fp8, causal, window, split)
    ("bf16", False, True, None, None), ("bf16", False, True, (63, 0), "plan"), ("reference", False, False, None, "4"),
    ("bf16", True, True, None, "plan"), ("bf16", True, True, (63, 0), None), ("reference", True, True, None, None),
    ("reference", True, False, (63, 0), "plan"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,fp8,causal,window,split", E2E)
def test_append_then_forward_equals_the_torch_recipe(mode, fp8, causal, window, split):
    """appendPagedKV then encode(paged=) gives O and L bit for bit those of the same forward over pools the torch
    recipe filled (index_copy_ at the slots; for FP8 the saturating quantization)."""
    _isolated("_check_end_to_end", mode, fp8, causal, window, split)


def _e2e_pools(mode, fp8, seed):
    """A decode and chunk step: queries / new tokens, the full keys, pools holding every key but the new ones (random
    filler there), and what the append writes"""
    from tests.test_paged_fp8_kv import quantize
    from tests.test_paged_kv import build_pool
    from tests.test_varlen import _descriptor, _inputs, _offsets
    rq, rk = [1, 1, 37, 0, 1], [1, 300, 90, 20, 1500]
    qo, ko = _offsets(rq), _offsets(rk)
    H, G, D = 8, 4, 128
    T, Tk = qo[-1] + 5, ko[-1]
    desc = _descriptor(T, Tk, D, mode, H, True)
    x = _inputs(desc, G, T, Tk, seed)
    scales = None
    if fp8:
        rng = np.random.default_rng(seed)
        scales = [(np.abs(x[op]).max(axis=(1, 2)) / 300 * rng.uniform(1.0, 1.3, H // G)).astype(np.float32)
                  for op in (Op.K, Op.V)]
    Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, 16, np.random.default_rng(seed))
    new = np.concatenate([np.arange(ko[s + 1] - rq[s], ko[s + 1]) for s in range(len(rq))]).astype(np.int64)
    slots = torch_slot_mapping(qo, rk, table, 16)
    for pool in (Kp, Vp):   # the new tokens' rows hold filler until the step writes them
        pool.reshape(-1, H // G, D)[slots] = np.random.default_rng(seed + 1).standard_normal((len(slots), H // G, D))
    k_new = np.zeros((T, H // G, D), np.float32)
    v_new = np.zeros((T, H // G, D), np.float32)
    k_new[:qo[-1]] = np.swapaxes(x[Op.K][:, new], 0, 1)
    v_new[:qo[-1]] = np.swapaxes(x[Op.V][:, new], 0, 1)
    if fp8:   # (the pools' other rows hold E4M3 values of the scaled keys, as a cache the append filled would)
        Kp = quantize(np.swapaxes(Kp.reshape(-1, H // G, D), 0, 1), scales[0]).swapaxes(0, 1).reshape(Kp.shape)
        Vp = quantize(np.swapaxes(Vp.reshape(-1, H // G, D), 0, 1), scales[1]).swapaxes(0, 1).reshape(Vp.shape)
    return desc, G, x, qo, rk, table, Kp, Vp, k_new, v_new, slots, scales


def _check_end_to_end(mode, fp8, causal, window, split):
    import torch
    from tests.test_paged_fp8_kv import Fp8PagedRun, _window
    from tests.test_paged_kv import _upload
    from tests.test_split_decode import SplitPagedRun, _same
    desc, G, x, qo, rk, table, Kp, Vp, k_new, v_new, slots, scales = _e2e_pools(mode, fp8, 5 + causal)
    desc.causal = causal
    prec = desc.memoryPrecisions[Op.K]
    split = None if split is None else mfa.SplitKV(*(() if split == "plan" else (int(split),)))
    with _window(window):
        runs = []
        for _ in range(2):
            if fp8:
                runs.append(Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, scales[0], scales[1], split=split))
            else:
                runs.append(SplitPagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, split=split))
        ours, recipe = runs
        kn, vn = _upload(k_new, prec), _upload(v_new, prec)
        mfa.appendPagedKV(ours.paged, mfa.PagedKVAppend(kn.data_ptr(), vn.data_ptr(), k_new.shape[0], 0, k_new.shape[1],
                                                        k_new.shape[2], Kp.shape[0] * Kp.shape[1], prec),
                          ours.k.data_ptr(), ours.v.data_ptr(),
                          fp8=ours.fp8 if fp8 else None)
        # the torch recipe: slot mapping on the device, index_copy_ (for FP8 the saturating quantization first)
        idx = torch.tensor(slots, device="cuda")
        T = qo[-1]
        for which, (new, pool) in enumerate(((kn, recipe.k), (vn, recipe.v))):
            rows = pool.view(-1, k_new.shape[1] * k_new.shape[2])
            src = new.view(torch.float16 if prec == P.FP16 else torch.bfloat16).view(k_new.shape[0], -1)[:T]
            if fp8:
                s = torch.from_numpy(scales[which]).cuda()
                q = (src.float().view(T, k_new.shape[1], -1) / s[None, :, None]).clamp(-E4M3_MAX, E4M3_MAX)
                src = q.to(torch.float8_e4m3fn).view(torch.uint8).view(T, -1)
            rows.index_copy_(0, idx, src.view(rows.dtype))
        torch.cuda.synchronize()
        assert torch.equal(ours.k, recipe.k) and torch.equal(ours.v, recipe.v)
        out = []
        for run in runs:
            run.encode()
            out.append(run.results())
    _same(*out)
    assert np.isfinite(out[0]["O"][:, :qo[-1]]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_captured_decode_step_replays_as_the_cache_grows(fp8):
    """One decode step (append, then the split forward) captured once and replayed for several steps while the test
    grows column_lengths and page_table on the device: each step's O, L and pools equal an eager step's bit for bit."""
    _isolated("_check_graph_replay", fp8)


def _check_graph_replay(fp8):
    import torch
    from tests.test_paged_fp8_kv import Fp8PagedRun
    from tests.test_paged_kv import build_pool, _upload
    from tests.test_split_decode import SplitPagedRun, _same
    from tests.test_varlen import _descriptor, _inputs, _offsets
    P_, H, G, D, steps = 16, 8, 4, 128, 6
    before = [1000, 300]
    final = [c + steps for c in before]
    qo = _offsets([1, 1])
    desc = _descriptor(2, 4096, D, "bf16", H, True)
    x = _inputs(desc, G, 2, sum(final), seed=41)
    ko = _offsets(final)
    Kp, Vp, table_final = build_pool(x[Op.K], x[Op.V], ko, P_, np.random.default_rng(41), spare_pages=4)
    for pool in (Kp, Vp):   # the keys the steps append hold filler until a step writes them
        slots = torch_slot_mapping(_offsets([steps] * 2), final, table_final, P_)
        pool.reshape(-1, H // G, D)[slots] = np.random.default_rng(42).standard_normal((len(slots), H // G, D))
    scales = [np.array([0.013, 0.021], np.float32), np.array([0.017, 0.011], np.float32)]

    def table_for(lengths):
        t = table_final.copy()
        for s, c in enumerate(lengths):
            t[s, -(-c // P_):] = -1
        return t

    def make():
        lengths = [c + 1 for c in before]
        if fp8:
            return Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, lengths, table_for(lengths), scales[0], scales[1],
                               split=mfa.SplitKV())
        return SplitPagedRun(desc, G, x[Op.Q], Kp, Vp, qo, lengths, table_for(lengths), split=mfa.SplitKV())

    graphed, eager = make(), make()
    assert graphed.plan().splits > 1
    news = [torch.zeros((2, H // G, D), dtype=torch.int16, device="cuda") for _ in range(2)]

    def step(run, stream=0):
        a = mfa.PagedKVAppend(news[0].data_ptr(), news[1].data_ptr(), 2, 0, H // G, D, Kp.shape[0] * P_, P.BF16)
        mfa.appendPagedKV(run.paged, a, run.k.data_ptr(), run.v.data_ptr(), fp8=run.fp8 if fp8 else None,
                          stream=stream)
        run.encode(stream)

    stream = torch.cuda.Stream()
    step(graphed, stream.cuda_stream)   # (outside any capture first, on the capturing stream: its workspace)
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        step(graphed, stream.cuda_stream)
    for n in range(steps):
        lengths = [c + 1 + n for c in before]
        for which, op in enumerate((Op.K, Op.V)):
            tokens = [ko[s] + lengths[s] - 1 for s in range(2)]
            news[which].copy_(_upload(np.ascontiguousarray(np.swapaxes(x[op][:, tokens], 0, 1)), P.BF16).view(2, H // G, D))
        for run in (graphed, eager):
            run.lengths.copy_(torch.tensor(lengths, dtype=torch.int32))
            run.table.copy_(torch.tensor(table_for(lengths), dtype=torch.int32))
            run.O.fill_(float("nan"))
            run.L.fill_(float("nan"))
        graph.replay()
        step(eager)
        _same(graphed.results(), eager.results())
        assert torch.equal(graphed.k, eager.k) and torch.equal(graphed.v, eager.v)
        assert np.isfinite(eager.results()["O"][:, :2]).all()
