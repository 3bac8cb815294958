"""Rotary append (appendPagedKV(..., rotary=Rotary(...))): the paged K/V append with the step's queries and new keys
rotated by RoPE at their cache positions, and the queries written in the paged forward's [H][rows][D] layout.

New token i of sequence s sits at position p = Cs - Rs + i, the key the plain append writes.  The reference rotates
op by op in torch on the CPU, (x.float() * c - y.float() * s).to(dtype), for the pairs (j, j + r/2) (GPT-NeoX) or
(2j, 2j + 1) (GPT-J), and maps slots as tests/test_paged_kv_append.py does.  On the GPU, q_out and both pools must equal
it byte for byte (NaN as NaN in FP8 pools), and every other byte, guard tails included, must keep its sentinel.  The
new call's buffers equal torch rope followed by the plain append, so the paged forward over them gives the same O and
L; a captured step replays as the cache grows."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import mfa_b200 as mfa
from tests.test_paged_kv_append import e4m3_reference

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ the reference
def pair_indices(r, interleaved):
    """the x and y elements of the r / 2 pairs"""
    return (slice(0, r, 2), slice(1, r, 2)) if interleaved else (slice(0, r // 2), slice(r // 2, r))


def rope(x, cos, sin, positions, r, interleaved):
    """x [N][heads][D] (any float torch dtype) rotated at positions [N]: cos / sin [positions][>= r/2] float32 tables.
    Op by op in float32, then rounded to x's dtype."""
    import torch
    pos = torch.as_tensor(np.asarray(positions, np.int64))
    c = torch.as_tensor(cos)[pos, :r // 2][:, None, :]
    s = torch.as_tensor(sin)[pos, :r // 2][:, None, :]
    xf = x.float()
    i1, i2 = pair_indices(r, interleaved)
    a, b = xf[..., i1], xf[..., i2]
    out = xf.clone()
    out[..., i1] = a * c - b * s
    out[..., i2] = b * c + a * s
    return out.to(x.dtype)


def rope_tables(positions, r, base=10000.0, seed=0):
    """cos, sin [positions][r/2] float32 of theta = p * base^(-2j/r), with a random phase per frequency so that the
    low positions exercise every quadrant too"""
    rng = np.random.default_rng(seed)
    inv = base ** (-np.arange(0, r, 2, dtype=np.float64) / r)
    theta = np.arange(positions, dtype=np.float64)[:, None] * inv[None, :] + rng.uniform(0, 2 * np.pi, r // 2)
    return np.cos(theta).astype(np.float32), np.sin(theta).astype(np.float32)


def token_positions(row_offsets, lengths, table, page_size, rows, pool_rows):
    """[(source token, position, pool row or None)] of every token the call rotates: position p >= 0; pool row None
    where the plain append skips the write (a page id outside the pool)"""
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
            out.append((lo + i, p, page * page_size + p % page_size if 0 <= page < pages else None))
    return out


# ------------------------------------------------------------------------------------------------ CPU: the API
def test_rotary_struct_and_version():
    assert ctypes.sizeof(mfa.Rotary) == 56
    offsets = {name: getattr(mfa.Rotary, name).offset for name, _ in mfa.Rotary._fields_}
    assert offsets == {"q_new": 0, "q_out": 8, "cos": 16, "sin": 24, "query_heads": 32, "q_token_stride": 36,
                       "rotary_dim": 40, "table_stride": 44, "positions": 48, "interleaved": 52}
    assert hasattr(mfa._lib, "mfa_paged_kv_append_rotary")
    v = mfa.version()
    assert "rotary append" in v and "paged K/V append" in v and "FP8 K/V" in v and " 0.5 " in v
    assert "Rotary" in mfa.__all__


def test_reference_rotation_is_the_formula():
    """The torch reference equals a NumPy float32 restatement of x' = x c - y s, y' = y c + x s, both pairings."""
    import torch
    rng = np.random.default_rng(3)
    N, Hd, D, r = 9, 3, 24, 16
    cos, sin = rope_tables(50, r, seed=3)
    pos = rng.integers(0, 50, N)
    x = rng.standard_normal((N, Hd, D)).astype(np.float32) * 3
    for interleaved in (False, True):
        got = rope(torch.from_numpy(x), cos, sin, pos, r, interleaved).numpy()
        want = x.copy()
        for j in range(r // 2):
            e0, e1 = (2 * j, 2 * j + 1) if interleaved else (j, j + r // 2)
            c, s = cos[pos, j][:, None], sin[pos, j][:, None]
            xa, ya = x[:, :, e0], x[:, :, e1]
            want[:, :, e0] = np.float32(xa * c) - np.float32(ya * s)
            want[:, :, e1] = np.float32(ya * c) + np.float32(xa * s)
        assert got.tobytes() == want.tobytes(), interleaved
        assert (got[:, :, r:] == x[:, :, r:]).all()


def _paged(S=2, max_row=4, rows=16, lengths=16, table=16, stride=4, page=16):
    return mfa.PagedKV(S, max_row, rows, lengths, table, stride, page)   # (device pointers are not dereferenced)


def _append(k=16, v=16, rows=8, stride=0, heads=2, D=64, pool_rows=256, prec=P.BF16):
    return mfa.PagedKVAppend(k, v, rows, stride, heads, D, pool_rows, prec)


def _rotary(q=16, out=16, cos=16, sin=16, H=4, stride=0, r=64, table_stride=0, positions=64, interleaved=0):
    return mfa.Rotary(q, out, cos, sin, H, stride, r, table_stride, positions, interleaved)


def _expect_error(call, message):
    with pytest.raises(mfa.MFAError) as e:
        call()
    assert e.value.status == -2 and message in e.value.message, e.value.message


def test_invalid_rotary_appends_are_rejected():
    """Each rejection names its field, before any device work (no GPU is needed to reach them)."""
    bad = [(_rotary(q=0), "Rotary append: q_new must not be NULL"),
           (_rotary(out=0), "Rotary append: q_out must not be NULL"),
           (_rotary(cos=0), "Rotary append: cos must not be NULL"),
           (_rotary(sin=0), "Rotary append: sin must not be NULL"),
           (_rotary(H=0), "query_heads 0 is not a positive multiple of kv_heads = 2"),
           (_rotary(H=3), "query_heads 3 is not a positive multiple of kv_heads = 2"),
           (_rotary(stride=255), "q_token_stride 255 is below query_heads * head_dimension = 256"),
           (_rotary(r=0), "rotary_dim 0 must be even and in [2, head_dimension = 64]"),
           (_rotary(r=63), "rotary_dim 63 must be even"),
           (_rotary(r=66), "rotary_dim 66 must be even and in [2, head_dimension = 64]"),
           (_rotary(r=64, table_stride=31), "table_stride 31 is below rotary_dim / 2 = 32"),
           (_rotary(positions=63), "positions 63 is below page_stride * page_size = 64"),
           (_rotary(interleaved=2), "interleaved 2 is not 0 or 1")]
    for rotary, message in bad:
        _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(), 16, 16, rotary=rotary), message)
        _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(), 16, 16, fp8=mfa.FP8KV(), rotary=rotary), message)
    # query_heads * D past 2^32 - 1 (only reachable with q_token_stride 0)
    _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(heads=1, D=512), 16, 16,
                                            rotary=_rotary(H=2**23 + 1, r=2)),
                  "query_heads * head_dimension = 4294967808 exceeds 2^32 - 1")
    # positions are compared with page_stride * page_size in 64 bits
    _expect_error(lambda: mfa.appendPagedKV(_paged(stride=2**30, page=16), _append(), 16, 16,
                                            rotary=_rotary(positions=2**32 - 1)),
                  "positions 4294967295 is below page_stride * page_size = 17179869184")
    err = mfa._lib.mfa_paged_kv_append_rotary(ctypes.byref(_paged()), ctypes.byref(_append()), None,
                                              ctypes.c_void_p(16), ctypes.c_void_p(16), None, None)
    assert err == -2 and "Rotary append: NULL rotary." in mfa._lib.mfa_last_error().decode()


def test_plain_append_messages_are_unchanged_through_the_rotary_call():
    """Every check of the plain append comes first, with its own words, whatever the rotary holds."""
    bad = [(None, _append(), "NULL paged K/V table"),
           (_paged(), None, "Paged K/V append: NULL append"),
           (_paged(), _append(k=0), "Paged K/V append: k_new must not be NULL"),
           (_paged(), _append(v=0), "Paged K/V append: v_new must not be NULL"),
           (_paged(rows=0), _append(), "row_offsets must not be NULL"),
           (_paged(S=0), _append(), "count 0 is outside [1, 65535]"),
           (_paged(max_row=9), _append(), "max_row 9 is outside [1, rows = 8]"),
           (_paged(page=24), _append(), "page_size 24 must be a power of two, at least 16, dividing pool_rows = 256"),
           (_paged(stride=0), _append(), "page_stride 0 must be at least 1"),
           (_paged(), _append(heads=0), "kv_heads 0 must be at least 1"),
           (_paged(), _append(D=513), "head_dimension 513 is outside [1, 512]"),
           (_paged(), _append(stride=127), "token_stride 127 is below kv_heads * head_dimension = 128"),
           (_paged(), _append(prec=3), "precision 3 is not MFA_FP32, MFA_FP16 or MFA_BF16")]
    for paged, append, message in bad:
        for rotary in (_rotary(), _rotary(q=0, r=3)):
            _expect_error(lambda: mfa.appendPagedKV(paged, append, 16, 16, rotary=rotary), message)
    _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(), 0, 16, rotary=_rotary(q=0)),
                  "Paged K/V append: k_pool must not be NULL")
    _expect_error(lambda: mfa.appendPagedKV(_paged(), _append(), 16, 0, rotary=_rotary(q=0)),
                  "Paged K/V append: v_pool must not be NULL")


def test_cpp_host_mirror_of_the_rotary_append(tmp_path):
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include <cstring>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  static int32_t fake[4];
  static float table[4];
  const PagedKV paged{1, 1, fake, fake, fake, 4, 16};
  const PagedKVAppend append{fake, fake, 1, 0, 2, 64, 64, MFA_BF16};
  const Rotary rotary{fake, fake, table, table, 4, 0, 63, 0, 64, 0};   // rotary_dim 63
  const FP8KV fp8{nullptr, nullptr};
  for (const FP8KV *f : {static_cast<const FP8KV *>(nullptr), &fp8}) {
    try {
      appendPagedKV(paged, append, rotary, fake, fake, f);
    } catch (const std::exception &e) {
      std::printf("%s\n", std::strstr(e.what(), "rotary_dim 63") ? "rejected" : e.what());
    }
  }
  std::printf("%zu\n", sizeof(Rotary));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    assert out[:3] == ["rejected", "rejected", "56"], out


def test_ptxas_rotary_kernels_have_no_spills_and_no_stack_frame():
    log = os.path.join(ROOT, "metal-flash-attention_b200", "_build", "kernels", "rotary_append.o.ptxas.log")
    assert os.path.exists(log), f"{log} is missing: build() writes it when it compiles the library"
    report, function = {}, None
    for line in open(log).read().splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            function = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and function is not None:
            report[function] = tuple(int(x) for x in m.groups())
            function = None
    kernels = {name: r for name, r in report.items() if "rotary_kv_append" in name}
    # FP32 / FP16 / BF16 sources x (copy, E4M3) x (NeoX, interleaved) x (vector, scalar)
    assert len(kernels) == 24, sorted(kernels)
    assert all(r == (0, 0, 0) for r in kernels.values()), kernels


# ------------------------------------------------------------------------------------------------ GPU
# Each GPU check runs in a process of its own: the launch-count tests of other suites record torch.profiler traces
# that are fragile to what ran before them in the same process.
def _isolated(check, *args):
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_rotary_append as t; "
            f"t.{check}(*{args!r})")
    proc = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]


TORCH_DTYPE = {"fp32": "float32", "fp16": "float16", "bf16": "bfloat16"}
PREC = {"fp32": P.FP32, "fp16": P.FP16, "bf16": P.BF16}
LENGTHS = {  # (new tokens Rs, cache lengths Cs with them)
    # decode, a chunk crossing pages with Cs - Rs not page-aligned, Rs = 0, a chunk starting at key 0, and a mix
    "mixed": ([1, 40, 0, 1, 300, 17], [1, 75, 33, 258, 300, 17 + 5]),
    "decode": ([1] * 7, [1, 2, 16, 17, 64, 257, 1000]),
    # Rs > Cs (the first tokens have p < 0), Cs = 0, and a decode row
    "short": ([5, 3, 1, 20], [2, 0, 40, 9]),
}


class RotaryCase:
    """Device buffers of one rotary append: a fused projection [rows][H + 2 Hkv][D] whose q / k / v are read in place
    (fused) or as contiguous copies; tables; cos / sin tables of page_stride * P positions (FlashAttention's [pos][r/2],
    or vLLM's cos_sin_cache [pos][r] through table_stride); q_out and both pools filled with random sentinel bytes plus
    a guard tail.  Source rows outside every sequence hold NaN."""

    def __init__(self, dtype, page_size, Hkv, G, D, r, interleaved, fused, table_mode, lengths, seed, fp8=None):
        import torch
        self.torch = torch
        rng = np.random.default_rng(seed)
        rq, rk = LENGTHS[lengths]
        self.P, self.Hkv, self.H, self.D, self.r, self.interleaved = page_size, Hkv, Hkv * G, D, r, interleaved
        self.qo = np.asarray([2] + list(2 + np.cumsum(rq)), np.int64)
        self.rows = int(self.qo[-1]) + 3   # (rows before the first and after the last sequence)
        pages_of = [-(-max(int(c), 0) // page_size) for c in rk]
        stride = max(1, max(pages_of))
        num_pages = sum(pages_of) + 4
        order = rng.permutation(num_pages)
        table = np.full((len(rk), stride), -1, np.int64)
        n = 0
        for s, count in enumerate(pages_of):
            table[s, :count] = order[n:n + count]
            n += count
        self.table_np, self.lengths_np, self.pool_rows = table, np.asarray(rk, np.int64), num_pages * page_size
        dt = getattr(torch, TORCH_DTYPE[dtype])
        self.dtype, self.prec = dt, PREC[dtype]
        H = self.H
        values = rng.standard_normal((self.rows, H + 2 * Hkv, D)).astype(np.float32) * 2
        if fp8 is not None:   # values past 448 after scaling: the quantization saturates
            big = rng.random(values.shape) < 0.02
            values[big] *= 400
        fused_t = torch.from_numpy(values).to(dt)
        inside = np.zeros(self.rows, bool)
        for s in range(len(rk)):
            inside[self.qo[s]:self.qo[s + 1]] = True
        fused_t[torch.from_numpy(~inside)] = float("nan")
        self.fused = fused_t.cuda()
        parts = (self.fused[:, :H], self.fused[:, H:H + Hkv], self.fused[:, H + Hkv:])
        if fused:
            self.q_new, self.k_new, self.v_new = parts
            self.q_stride = self.token_stride = (H + 2 * Hkv) * D
        else:
            self.q_new, self.k_new, self.v_new = (x.contiguous() for x in parts)
            self.q_stride = self.token_stride = 0
        self.positions = stride * page_size
        self.cos, self.sin = rope_tables(self.positions, r, seed=seed)
        if table_mode == "vllm":
            cache = np.concatenate([self.cos, self.sin], axis=1)   # [pos][r]: cos half, then sin half
            self.table_dev = torch.from_numpy(cache).cuda()
            cos_ptr = self.table_dev.data_ptr()
            sin_ptr = cos_ptr + 4 * (r // 2)
            table_stride = r
        else:
            self.cos_dev, self.sin_dev = torch.from_numpy(self.cos).cuda(), torch.from_numpy(self.sin).cuda()
            cos_ptr, sin_ptr, table_stride = self.cos_dev.data_ptr(), self.sin_dev.data_ptr(), 0
        self.fp8 = fp8
        esize = fused_t.element_size()
        self.row_bytes = Hkv * D * (1 if fp8 is not None else esize)
        self.q_row_bytes = D * esize
        g = torch.Generator(device="cuda")
        g.manual_seed(seed)
        guard = 7
        self.k_pool, self.v_pool = (torch.randint(0, 256, ((self.pool_rows + guard) * self.row_bytes,),
                                                  dtype=torch.uint8, device="cuda", generator=g) for _ in range(2))
        self.q_out = torch.randint(0, 256, ((H * self.rows + guard) * self.q_row_bytes,), dtype=torch.uint8,
                                   device="cuda", generator=g)
        self.before = [b.clone() for b in (self.q_out, self.k_pool, self.v_pool)]
        self.row_offsets = torch.tensor(self.qo, dtype=torch.int32, device="cuda")
        self.lengths = torch.tensor(self.lengths_np, dtype=torch.int32, device="cuda")
        self.table = torch.tensor(table, dtype=torch.int32, device="cuda")
        max_row = max(1, int(np.max(np.diff(self.qo))))
        self.paged = mfa.PagedKV(len(rk), max_row, self.row_offsets.data_ptr(), self.lengths.data_ptr(),
                                 self.table.data_ptr(), stride, page_size)
        self.scales, self.fp8_arg = None, None
        if fp8 is not None:
            self.scales = [None if s is None else torch.tensor(np.asarray(s, np.float32), device="cuda") for s in fp8]
            self.fp8_arg = mfa.FP8KV(*(0 if s is None else s.data_ptr() for s in self.scales))
        self.rotary = mfa.Rotary(self.q_new.data_ptr(), self.q_out.data_ptr(), cos_ptr, sin_ptr, H, self.q_stride, r,
                                 table_stride, self.positions, int(interleaved))

    def append(self):
        a = mfa.PagedKVAppend(self.k_new.data_ptr(), self.v_new.data_ptr(), self.rows, self.token_stride, self.Hkv,
                              self.D, self.pool_rows, self.prec)
        mfa.appendPagedKV(self.paged, a, self.k_pool.data_ptr(), self.v_pool.data_ptr(), fp8=self.fp8_arg,
                          rotary=self.rotary)

    def check(self):
        """q_out rows of tokens with p >= 0 hold rope(q); the pool rows the plain append names hold rope(k) and v (FP8:
        quantized, NaN as NaN); every other byte keeps its sentinel"""
        torch = self.torch
        torch.cuda.synchronize()
        rotated = token_positions(self.qo, self.lengths_np, self.table_np, self.P, self.rows, self.pool_rows)
        q_before, k_before, v_before = (b.cpu() for b in self.before)
        expected_q = q_before.clone()
        if rotated:
            tokens = [t for t, _, _ in rotated]
            pos = [p for _, p, _ in rotated]
            q = rope(self.q_new[tokens].cpu(), self.cos, self.sin, pos, self.r, self.interleaved)
            region = expected_q[:self.H * self.rows * self.q_row_bytes].view(self.H, self.rows, self.q_row_bytes)
            region[:, tokens] = q.contiguous().view(torch.uint8).view(len(tokens), self.H, -1).transpose(0, 1)
        got_q = self.q_out.cpu()
        diff = (expected_q != got_q).view(-1, self.q_row_bytes).any(dim=1).nonzero().flatten().tolist()
        assert not diff, f"q_out rows differ from the reference: {diff[:10]} ({len(rotated)} tokens rotated)"
        written = [(t, p, row) for t, p, row in rotated if row is not None]
        for which, (src, after, before) in enumerate(((self.k_new, self.k_pool, k_before),
                                                      (self.v_new, self.v_pool, v_before))):
            expected = before.clone().view(-1, self.row_bytes)
            got = after.cpu().view(-1, self.row_bytes)
            if written:
                x = src[[t for t, _, _ in written]].cpu()
                if which == 0:
                    x = rope(x, self.cos, self.sin, [p for _, p, _ in written], self.r, self.interleaved)
                rows = torch.tensor([row for _, _, row in written])
                if self.fp8 is None:
                    want = x.contiguous().view(torch.uint8).reshape(len(written), self.row_bytes)
                else:
                    want = e4m3_reference(x, self.fp8[which]).reshape(len(written), self.row_bytes)
                    nan = (want & 0x7F) == 0x7F
                    have = got[rows]
                    assert ((have[nan] & 0x7F) == 0x7F).all(), "NaN stays NaN"
                    want = torch.where(nan, have, want)
                expected[rows] = want
            diff = (expected != got).any(dim=1).nonzero().flatten().tolist()
            assert not diff, f"{'KV'[which]} pool rows differ from the reference: {diff[:10]} ({len(written)} written)"
        return rotated, written


EXACT_CASES = [  # (dtype, P, Hkv, G, D, r, interleaved, fused, table, fp8: None / "scaled" / "null")
    ("bf16", 16, 8, 4, 128, 128, 0, False, "flash", None),
    ("bf16", 64, 2, 8, 128, 64, 1, True, "vllm", None),
    ("fp16", 256, 1, 1, 64, 64, 1, False, "flash", None),
    ("fp16", 16, 2, 4, 80, 80, 0, True, "flash", None),
    ("fp32", 64, 1, 4, 40, 40, 0, False, "flash", None),
    ("bf16", 64, 8, 1, 256, 128, 0, False, "vllm", None),
    ("bf16", 16, 2, 4, 64, 2, 0, False, "flash", None),      # r = 2: the scalar path
    ("fp16", 64, 1, 8, 128, 2, 1, True, "flash", None),
    ("bf16", 16, 2, 4, 128, 24, 0, False, "flash", None),    # r / 2 = 12, not a multiple of 8: scalar
    ("fp32", 16, 2, 1, 64, 36, 1, False, "vllm", None),      # r / 2 = 18, not a multiple of 4: scalar
    ("bf16", 256, 2, 4, 40, 20, 1, True, "flash", None),
    ("bf16", 16, 8, 4, 128, 128, 0, False, "flash", "scaled"),
    ("bf16", 64, 2, 4, 128, 64, 1, True, "vllm", "null"),
    ("fp16", 16, 1, 8, 64, 32, 0, False, "flash", "scaled"),
    ("fp32", 64, 2, 4, 80, 80, 1, False, "flash", "scaled"),
    ("bf16", 256, 1, 1, 256, 256, 0, True, "flash", "null"),
    ("fp16", 16, 2, 4, 80, 80, 0, False, "flash", "scaled"),  # r / 2 = 40, not a multiple of 16: scalar E4M3
    ("bf16", 64, 8, 1, 64, 2, 1, False, "vllm", "scaled"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_rotary_appends_write_exactly_the_reference_rows(fp8):
    """Both pairings, r = D, D/2, 2 and widths that force the scalar path, D 40..256, BF16 / FP16 / FP32, Hkv 1/2/8,
    G 1/4/8, P 16/64/256, fused sources, vLLM's cos_sin_cache, FP8 pools with arbitrary and NULL scales, decode and
    chunk rows, empty sequences and Rs > Cs: q_out and the pools equal the reference byte for byte, every other byte
    keeps its sentinel."""
    _isolated("_check_cases", [c for c in EXACT_CASES if (c[9] is not None) == fp8])


def _check_cases(cases):
    for n, case in enumerate(cases):
        dtype, P_, Hkv, G, D, r, interleaved, fused, table, fp8 = case
        for lengths in LENGTHS:
            seed = 100 * n + len(lengths)
            scales = None
            if fp8 == "scaled":
                rng = np.random.default_rng(seed)
                scales = tuple((rng.uniform(0.05, 3.0, Hkv) * (1 + 1 / 3)).astype(np.float32) for _ in range(2))
            elif fp8 == "null":
                scales = (None, None)
            c = RotaryCase(dtype, P_, Hkv, G, D, r, interleaved, fused, table, lengths, seed, fp8=scales)
            c.append()
            rotated, written = c.check()
            rq, rk = LENGTHS[lengths]
            assert len(written) == len(rotated) == sum(min(q, max(k, 0)) for q, k in zip(rq, rk)), (case, lengths)


# ------------------------------------------------------------------------------------------------ GPU: end to end
E2E = [  # (mode, fp8, causal, window, split, r, interleaved)
    ("bf16", False, True, None, None, 128, 0), ("bf16", False, True, (63, 0), "plan", 64, 1),
    ("fp16", False, False, None, "4", 128, 1), ("bf16", True, True, None, "plan", 128, 0),
    ("bf16", True, True, (63, 0), None, 64, 0), ("fp16", True, False, (63, 0), "plan", 128, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,fp8,causal,window,split,r,interleaved", E2E)
def test_rotary_append_then_forward_equals_the_torch_recipe(mode, fp8, causal, window, split, r, interleaved):
    """The rotary append's Q and pools equal torch rope, the transpose and appendPagedKV bit for bit, so the paged
    forward over them gives the same O and L; the 16-bit runs also match the float64 reference attention over the
    rotated queries and keys."""
    _isolated("_check_end_to_end", mode, fp8, causal, window, split, r, interleaved)


def _check_end_to_end(mode, fp8, causal, window, split, r, interleaved):
    import torch
    from tests.test_paged_fp8_kv import Fp8PagedRun, _window
    from tests.test_paged_kv import _upload
    from tests.test_paged_kv_append import _e2e_pools
    from tests.test_split_decode import SplitPagedRun, _same
    from tests.test_varlen import _offsets, reference
    desc, G, x, qo, rk, table, Kp, Vp, k_new, v_new, slots, scales = _e2e_pools(mode, fp8, 9 + causal)
    desc.causal = causal
    prec = desc.memoryPrecisions[Op.K]
    assert desc.memoryPrecisions[Op.Q] == prec
    dt = torch.float16 if prec == P.FP16 else torch.bfloat16
    H, T, D = x[Op.Q].shape
    Hkv = H // G
    positions = table.shape[1] * 16
    cos, sin = rope_tables(positions, r, seed=5)
    cos_dev, sin_dev = torch.from_numpy(cos).cuda(), torch.from_numpy(sin).cuda()
    split = None if split is None else mfa.SplitKV(*(() if split == "plan" else (int(split),)))
    q_new = _upload(np.ascontiguousarray(np.swapaxes(x[Op.Q], 0, 1)), prec)   # [T][H][D], before rotation
    kn, vn = _upload(k_new, prec), _upload(v_new, prec)
    with _window(window):
        runs = []
        for _ in range(2):
            if fp8:
                runs.append(Fp8PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, scales[0], scales[1], split=split))
            else:
                runs.append(SplitPagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table, split=split))
        ours, recipe = runs
        append = mfa.PagedKVAppend(kn.data_ptr(), vn.data_ptr(), T, 0, Hkv, D, Kp.shape[0] * Kp.shape[1], prec)
        mfa.appendPagedKV(ours.paged, append, ours.k.data_ptr(), ours.v.data_ptr(), fp8=ours.fp8 if fp8 else None,
                          rotary=mfa.Rotary(q_new.data_ptr(), ours.q.data_ptr(), cos_dev.data_ptr(),
                                            sin_dev.data_ptr(), H, 0, r, 0, positions, interleaved))
        # the torch recipe: positions from the device tables, rope on q and k, the transpose, then the plain append
        n = int(qo[-1])
        offsets = recipe.rows.long()
        Rs = torch.diff(offsets)
        seq = torch.repeat_interleave(torch.arange(len(rk), device="cuda"), Rs, output_size=n)
        pos = recipe.lengths.long()[seq] - Rs[seq] + torch.arange(n, device="cuda") - offsets[seq]
        qr = rope_device(q_new.view(dt)[:n], cos_dev, sin_dev, pos, r, interleaved)
        kr = kn.view(dt).view(T, Hkv, D).clone()
        kr[:n] = rope_device(kr[:n], cos_dev, sin_dev, pos, r, interleaved)
        recipe.q.view(dt).view(H, T, D)[:, :n] = qr.transpose(0, 1)
        mfa.appendPagedKV(recipe.paged, mfa.PagedKVAppend(kr.data_ptr(), vn.data_ptr(), T, 0, Hkv, D,
                                                          Kp.shape[0] * Kp.shape[1], prec),
                          recipe.k.data_ptr(), recipe.v.data_ptr(), fp8=recipe.fp8 if fp8 else None)
        torch.cuda.synchronize()
        assert torch.equal(ours.q, recipe.q), "Q"
        assert torch.equal(ours.k, recipe.k) and torch.equal(ours.v, recipe.v), "pools"
        out = []
        for run in runs:
            run.encode()
            out.append(run.results())
    _same(*out)
    assert np.isfinite(out[0]["O"][:, :n]).all()
    if not fp8 and window is None:   # the float64 reference over the rotated queries and the cache with rotated keys
        K = x[Op.K].copy()
        ko = _offsets(rk)
        new = np.concatenate([np.arange(ko[s + 1] - (qo[s + 1] - qo[s]), ko[s + 1]) for s in range(len(rk))])
        K[:, new] = kr[:n].float().cpu().numpy().swapaxes(0, 1)
        Q = np.zeros_like(x[Op.Q])
        Q[:, :n] = qr.float().cpu().numpy().swapaxes(0, 1)
        ref = reference({Op.Q: Q, Op.K: K, Op.V: x[Op.V], Op.dO: np.zeros_like(Q)}, G, qo, ko, causal)
        errO = float(np.abs(out[0]["O"][:, :n] - ref["O"][:, :n]).max())
        errL = float(np.abs(out[0]["L"][:, :n] / 1.44269504089 - ref["L"][:, :n]).max())
        assert errO < 2e-2 and errL < 1e-3, (errO, errL)


def rope_device(x, cos, sin, pos, r, interleaved):
    """rope on device tensors: x [N][heads][D], pos [N] int64 on the device; op by op in float32"""
    c = cos[pos, :r // 2][:, None, :]
    s = sin[pos, :r // 2][:, None, :]
    xf = x.float()
    i1, i2 = pair_indices(r, interleaved)
    a, b = xf[..., i1], xf[..., i2]
    out = xf.clone()
    out[..., i1] = a * c - b * s
    out[..., i2] = b * c + a * s
    return out.to(x.dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_captured_rotary_step_replays_as_the_cache_grows(fp8):
    """One decode step (rotary append, then the split forward) captured once and replayed for several steps while the
    test grows column_lengths and page_table on the device: each step's O, L, Q and pools equal an eager step's bit
    for bit."""
    _isolated("_check_graph_replay", fp8)


def _check_graph_replay(fp8):
    import torch
    from tests.test_paged_fp8_kv import Fp8PagedRun
    from tests.test_paged_kv import build_pool, _upload
    from tests.test_paged_kv_append import torch_slot_mapping
    from tests.test_split_decode import SplitPagedRun, _same
    from tests.test_varlen import _descriptor, _inputs, _offsets
    P_, H, G, D, r, steps = 16, 8, 4, 128, 128, 6
    before = [1000, 300]
    final = [c + steps for c in before]
    qo = _offsets([1, 1])
    desc = _descriptor(2, 4096, D, "bf16", H, True)
    x = _inputs(desc, G, 2, sum(final), seed=43)
    ko = _offsets(final)
    Kp, Vp, table_final = build_pool(x[Op.K], x[Op.V], ko, P_, np.random.default_rng(43), spare_pages=4)
    for pool in (Kp, Vp):   # the keys the steps append hold filler until a step writes them
        slots = torch_slot_mapping(_offsets([steps] * 2), final, table_final, P_)
        pool.reshape(-1, H // G, D)[slots] = np.random.default_rng(44).standard_normal((len(slots), H // G, D))
    scales = [np.array([0.013, 0.021], np.float32), np.array([0.017, 0.011], np.float32)]
    positions = table_final.shape[1] * P_
    cos, sin = (torch.from_numpy(t).cuda() for t in rope_tables(positions, r, seed=6))

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
    news = [torch.zeros((2, n, D), dtype=torch.int16, device="cuda") for n in (H, H // G, H // G)]

    def step(run, stream=0):
        a = mfa.PagedKVAppend(news[1].data_ptr(), news[2].data_ptr(), 2, 0, H // G, D, Kp.shape[0] * P_, P.BF16)
        rot = mfa.Rotary(news[0].data_ptr(), run.q.data_ptr(), cos.data_ptr(), sin.data_ptr(), H, 0, r, 0, positions,
                         0)
        mfa.appendPagedKV(run.paged, a, run.k.data_ptr(), run.v.data_ptr(), fp8=run.fp8 if fp8 else None,
                          stream=stream, rotary=rot)
        run.encode(stream)

    stream = torch.cuda.Stream()
    step(graphed, stream.cuda_stream)   # (outside any capture first, on the capturing stream: its workspace)
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        step(graphed, stream.cuda_stream)
    rng = np.random.default_rng(45)
    for n in range(steps):
        lengths = [c + 1 + n for c in before]
        tokens = [ko[s] + lengths[s] - 1 for s in range(2)]
        q = rng.standard_normal((2, H, D)).astype(np.float32)
        news[0].copy_(torch.from_numpy(q).to(torch.bfloat16).view(torch.int16))
        for which, op in enumerate((Op.K, Op.V)):
            news[which + 1].copy_(_upload(np.ascontiguousarray(np.swapaxes(x[op][:, tokens], 0, 1)),
                                          P.BF16).view(2, H // G, D))
        for run in (graphed, eager):
            run.lengths.copy_(torch.tensor(lengths, dtype=torch.int32))
            run.table.copy_(torch.tensor(table_for(lengths), dtype=torch.int32))
            run.q.fill_(-1)
            run.O.fill_(float("nan"))
            run.L.fill_(float("nan"))
        graph.replay()
        step(eager)
        _same(graphed.results(), eager.results())
        assert torch.equal(graphed.q, eager.q)
        assert torch.equal(graphed.k, eager.k) and torch.equal(graphed.v, eager.v)
        assert np.isfinite(eager.results()["O"][:, :2]).all()
