"""Grouped-head decode tiles: the split-KV forward of packed and paged calls (and every FP8 call) packs the G query
heads of one K/V head into one tile when 2 <= G <= 128 and max_row < 128, m = floor(128 / G) query rows of each head.

The suites of the split and FP8 paths run G in {1, 4, 8}, where G * m = 128 and m is a multiple of 8.  Here every G
from 2 to 128 runs, with 256 as the one-head-per-tile fallback: groups that leave tile rows G * m .. 127 unloaded,
head sub-boxes of the Q box {64, m, G} that start off a 1024-byte swizzle period (m % 8 != 0), row maps with an m that
is not a power of two, FP16 L (lowPrecisionIntermediates) through the direct store of one split and through the merge
of several, and per-K/V-head FP8 scales with three K/V heads.

Each case checks O and L against the float64 reference (and the exact empty-row and sentinel bit patterns), a plan of
one split against the unsplit call with one head per tile bit for bit, the paged call against the packed call for the
same num_splits bit for bit, the query heads reversed inside every K/V group against the outputs reversed the same
way, FP8 against the 16-bit call on the dequantized pools, two runs over a workspace left full of stale partials, and
(windowed paged calls) pages outside the band pointing at a NaN page."""
import json
import os

import numpy as np
import pytest

import mfa_b200 as mfa
from tests.test_feature_matrix import _check_within, storage_error
from tests.test_paged_fp8_kv import Fp8PagedRun, dequantize, quantize
from tests.test_paged_kv import _check_sentinels, build_pool, run_packed_forward
from tests.test_split_decode import SplitPagedRun, _same, expected_plan, run_packed_split, run_paged_plain, \
    run_paged_split
from tests.test_varlen import LOG2E, _constants, _descriptor, _inputs, _offsets, reference
from tests.test_window import band_mask, band_reference

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision

MASKS = {"none": (False, None), "causal": (True, None), "window": (True, (63, 0)), "band": (False, (40, 20))}
GROUPS = [2, 3, 5, 6, 7, 12, 16, 24, 32, 48, 64, 100, 128]

# (form, operands, D, G, mask, FP16 L, num_splits (0: the plan), page size, lengths).  Forms: "packed" and "paged"
# split calls, "fp8" (NULL scales) and "fp8_scaled" (three K/V heads with distinct scales).  Each G in GROUPS has one
# case of each form: packed with SplitKV(1) (the direct store), paged with 3 or 16 splits (the merge); D = 64 and 256
# for every G with m % 8 != 0; four masks and two L formats in rotation.  Then the fallbacks (max_row = 128, G = 256),
# staged operands, library plans and a one-split paged call.
CASES = [
    ("packed", "bf16", 128, 2, "none", True, 1, 16, "edges"),
    ("paged", "fp16", 96, 2, "causal", False, 3, 64, "edges"),
    ("fp8", "reference", 64, 2, "window", True, 16, 256, "decode"),
    ("packed", "fp16", 64, 3, "causal", False, 1, 64, "edges"),
    ("paged", "reference", 256, 3, "window", True, 16, 256, "edges"),
    ("fp8_scaled", "bf16", 96, 3, "band", False, 0, 16, "edges"),
    ("packed", "reference", 64, 5, "window", True, 1, 256, "edges"),
    ("paged", "bf16", 256, 5, "band", False, 3, 16, "edges"),
    ("fp8", "fp16", 128, 5, "none", True, 3, 64, "decode"),
    ("packed", "bf16", 64, 6, "band", False, 1, 16, "edges"),
    ("paged", "fp16", 256, 6, "none", True, 16, 64, "edges"),
    ("fp8_scaled", "reference", 96, 6, "causal", False, 1, 256, "edges"),
    ("packed", "fp16", 64, 7, "none", True, 1, 64, "edges"),
    ("paged", "reference", 256, 7, "causal", False, 3, 256, "edges"),
    ("fp8", "bf16", 128, 7, "window", True, 16, 16, "decode"),
    ("packed", "reference", 64, 12, "causal", False, 1, 256, "edges"),
    ("paged", "bf16", 256, 12, "window", True, 3, 16, "edges"),
    ("fp8_scaled", "fp16", 96, 12, "band", False, 0, 64, "edges"),
    ("packed", "bf16", 128, 16, "window", True, 1, 16, "edges"),
    ("paged", "fp16", 96, 16, "band", False, 16, 64, "edges"),
    ("fp8", "reference", 64, 16, "none", True, 3, 256, "decode"),
    ("packed", "fp16", 64, 24, "band", False, 1, 64, "edges"),
    ("paged", "reference", 256, 24, "none", True, 3, 256, "edges"),
    ("fp8_scaled", "bf16", 128, 24, "causal", True, 16, 16, "edges"),
    ("packed", "reference", 64, 32, "none", True, 1, 256, "edges"),
    ("paged", "bf16", 256, 32, "causal", False, 16, 16, "edges"),
    ("fp8", "fp16", 96, 32, "window", True, 3, 64, "decode"),
    ("packed", "bf16", 64, 48, "causal", False, 1, 16, "edges"),
    ("paged", "fp16", 256, 48, "window", True, 3, 64, "edges"),
    ("fp8_scaled", "reference", 128, 48, "band", False, 1, 256, "edges"),
    ("packed", "fp16", 64, 64, "window", True, 1, 64, "edges"),
    ("paged", "reference", 256, 64, "band", False, 16, 256, "edges"),
    ("fp8", "bf16", 96, 64, "none", True, 3, 16, "decode"),
    ("packed", "reference", 64, 100, "band", False, 1, 256, "edges"),
    ("paged", "bf16", 256, 100, "none", True, 3, 16, "edges"),
    ("fp8", "fp16", 128, 100, "causal", False, 0, 64, "decode"),
    ("packed", "bf16", 64, 128, "none", True, 1, 16, "edges"),
    ("paged", "fp16", 256, 128, "causal", False, 16, 64, "edges"),
    ("fp8", "reference", 96, 128, "window", True, 3, 256, "decode"),
    # a windowed paged call with m = 1 (its pages outside the band point at a NaN page)
    ("paged", "bf16", 64, 128, "window", False, 3, 16, "decode"),
    # max_row = 128: one head per tile, split and FP16 L through the merge, or the plan
    ("paged", "bf16", 128, 7, "causal", True, 3, 16, "full"),
    ("packed", "fp16", 128, 7, "none", False, 0, 64, "full"),
    # G = 256: more query heads than tile rows, one head per tile
    ("packed", "bf16", 128, 256, "causal", True, 3, 16, "decode"),
    ("paged", "reference", 64, 256, "window", False, 1, 64, "decode"),
    ("fp8", "fp16", 256, 256, "none", True, 16, 256, "decode"),
    # staged operands (D = 60: Q, K, V staged with 64 columns, O copied back) around packed heads
    ("packed", "bf16", 60, 7, "causal", True, 3, 16, "edges"),
    ("packed", "reference", 60, 100, "window", False, 1, 16, "edges"),
    # the library's plan over long contexts, and one split on a paged call (against the unsplit paged call)
    ("paged", "bf16", 128, 24, "none", False, 0, 16, "decode"),
    ("packed", "fp16", 96, 5, "causal", True, 0, 16, "decode"),
    ("paged", "fp16", 128, 6, "window", True, 1, 16, "decode"),
    ("paged", "reference", 96, 12, "band", True, 1, 64, "edges"),
]


def tile_rows(G):
    """m: query rows of each head in a tile with packed heads (128: one head per tile)"""
    return 128 // G if 2 <= G <= 128 else 128


def case_id(case):
    form, mode, D, G, mask, low, n, page, profile = case
    return f"G{G}-m{tile_rows(G)}-{form}-{mode}-D{D}-{mask}-{'fp16L' if low else 'fp32L'}-split{n}-P{page}-{profile}"


def kv_heads(case):
    form, G = case[0], case[3]
    return 3 if form == "fp8_scaled" else (1 if G >= 64 else 2)


def case_lengths(profile, G, D):
    """(query lengths Rs, key lengths Cs) of the sequences.  edges: Rs at the tile edges of G (0, 1, m - 1, m, m + 1,
    2m + 1, at most 127, and 127), each with its own Cs so that delta = Cs - Rs differs: no key, one key, BN +- 1 and
    a long context among them.  decode: one row each over 0, 1, BN +- 1 and a long context, and a sequence without
    rows.  full: max_row = 128, so the plan keeps one head per tile."""
    BN = 64 if D > 128 else 128
    m = tile_rows(G)
    long = 3000 if G < 64 else 300
    if profile == "decode":
        return [1, 1, 1, 1, 1, 0], [0, 1, BN - 1, BN + 1, long, 7]
    if profile == "full":
        return [128, 1, 40], [200, long, 0]
    return [0, 1, m - 1, m, m + 1, min(2 * m + 1, 127), 127], [5, 0, BN - 1, BN + 1, long, 1, 2 * BN + 3]


def reversed_heads(H, G):
    """The query heads in reverse order inside every K/V group: new head h is old head perm[h]."""
    return np.array([g * G + G - 1 - i for g in range(H // G) for i in range(G)])


def band_poisoned_table(table, rq, rk, page_size, window, causal, nan_page):
    """A copy of the page table in which every page wholly outside the band of all of its sequence's rows points at
    nan_page or far outside the pool (alternately), as in tests/test_window.py; and the count of such entries."""
    left, right = window[0], 0 if causal else window[1]
    poisoned, n = table.copy(), 0
    for s, (Rs, Cs) in enumerate(zip(rq, rk)):
        delta = Cs - Rs
        lo, hi = delta - left, Rs - 1 + delta + right   # the lowest and highest key any row sees
        for j in range(-(-Cs // page_size)):
            if (j + 1) * page_size <= lo or j * page_size > hi:
                poisoned[s, j] = nan_page if n % 2 == 0 else 2**31 - 1
                n += 1
    return poisoned, n


class Case:
    """The inputs of one case: descriptor, float inputs, offsets, pools and page table (16-bit forms)."""

    def __init__(self, form, mode, D, G, mask, low, n, page, profile):
        self.form, self.mode, self.D, self.G, self.n, self.page = form, mode, D, G, n, page
        self.causal, self.window = MASKS[mask]
        self.Hkv = kv_heads((form, mode, D, G))
        self.H = G * self.Hkv
        self.rq, self.rk = case_lengths(profile, G, D)
        self.qo, self.ko = _offsets(self.rq), _offsets(self.rk)
        self.T, self.Tk = self.qo[-1] + 9, self.ko[-1] + 5   # rows past the table's end keep their sentinels
        self.seed = D + G + page + n
        self.desc = _descriptor(self.T, self.Tk, D, mode, self.H, self.causal, lowMid=low)
        self.x = _inputs(self.desc, G, self.T, self.Tk, self.seed)
        self.Kp, self.Vp, self.table = build_pool(self.x[Op.K], self.x[Op.V], self.ko, page,
                                                  np.random.default_rng(self.seed))
        self.split = mfa.SplitKV(n)

    def kernel(self):
        kd = self.desc.kernelDescriptor(KT.forward)
        return kd, mfa.AttentionKernel(kd, window=self.window) if self.window else mfa.AttentionKernel(kd)

    def plans(self):
        """(splitPlan of the case's call from host values, the documented rule's plan)"""
        kd, kernel = self.kernel()
        S, max_row = len(self.rq), max(1, max(self.rq))
        if self.form == "packed":
            c, layout = _constants(self.T, self.Tk, self.H, self.G), "sequences"
            table = mfa.SequenceTable(S, max_row, max(1, max(self.rk)), 16, 16)   # (not dereferenced on the host)
        else:
            c, layout = _constants(self.T, self.Kp.shape[0] * self.page, self.H, self.G), "paged"
            table = mfa.PagedKV(S, max_row, 16, 16, 16, self.table.shape[1], self.page)
        got = kernel.splitPlan(c, split=self.split, **{layout: table})
        staged = 4 if self.D % 8 and self.form == "packed" else 0
        want = expected_plan(kernel, c, table, self.split, kd.splitPolicy, window=self.window, staged=staged)
        return (got.splits, got.heads_per_tile, got.grid_size, got.launch_count), want

    def reference(self, x):
        inputs = {Op.Q: x[Op.Q], Op.K: x[Op.K], Op.V: x[Op.V], Op.dO: np.zeros_like(x[Op.Q])}
        if self.window is None:
            return reference(inputs, self.G, self.qo, self.ko, self.causal)
        return band_reference(inputs, self.G, self.qo, self.ko, self.window[0], 0 if self.causal else self.window[1])


# ------------------------------------------------------------------------------------------------ CPU
def test_the_case_list_covers_every_group():
    ids = [case_id(c) for c in CASES]
    assert len(set(ids)) == len(ids) and 40 <= len(CASES) <= 60, len(CASES)
    packed_heads = {G for G in GROUPS if 128 % G or tile_rows(G) % 8}
    assert packed_heads == {3, 5, 6, 7, 12, 24, 32, 48, 64, 100, 128}
    plans = {c: Case(*c).plans()[0] for c in CASES}
    for G in GROUPS + [256]:
        mine = [c for c in CASES if c[3] == G]
        assert {c[0] for c in mine} >= {"packed", "paged"} and {c[0] for c in mine} & {"fp8", "fp8_scaled"}, G
        if G == 256:
            assert all(plans[c][1] == 1 for c in mine)
            continue
        tiled = [c for c in mine if plans[c][1] == G]   # the cases whose tiles hold the group's heads
        assert {c[0] for c in tiled} >= {"packed", "paged"}, G
        assert any(c[5] for c in tiled), f"G = {G}: FP16 L"
        assert any(c[4] != "none" for c in tiled), f"G = {G}: a mask"
        assert any(plans[c][0] == 1 for c in tiled) and any(plans[c][0] > 1 for c in tiled), f"G = {G}: splits"
        assert any(c[6] == 1 for c in tiled), f"G = {G}: SplitKV(1)"
        if G in packed_heads:
            assert {c[2] for c in tiled} >= {64, 256}, f"G = {G}: D = 64 and 256"
    # FP16 L through the direct store and through the merge, on 16-bit and FP8 pools
    low = [plans[c][0] for c in CASES if c[5] and plans[c][1] > 1]
    assert 1 in low and max(low) > 1
    assert any(c[0] == "fp8" and c[5] and plans[c][0] > 1 and plans[c][1] > 1 for c in CASES)
    # distinct per-K/V-head FP8 scales under packed heads, with at least three K/V heads
    assert sum(1 for c in CASES if c[0] == "fp8_scaled" and plans[c][1] > 1 and kv_heads(c) >= 3) >= 4
    # a windowed paged case whose pages outside the band are poisoned, for m % 8 != 0 and for m = 1
    windowed_paged = [c for c in CASES if c[0] == "paged" and c[4] in ("window", "band") and plans[c][1] > 1]
    assert any(tile_rows(c[3]) % 8 for c in windowed_paged) and any(tile_rows(c[3]) == 1 for c in windowed_paged)
    # the fallback of max_row = 128, and every other case with max_row < 128
    assert any(c[8] == "full" and plans[c][1] == 1 and 2 <= c[3] <= 128 for c in CASES)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_split_plan_follows_the_rule(case):
    s = Case(*case)
    got, want = s.plans()
    assert got == want, (got, want)
    assert got[1] == (s.G if 2 <= s.G <= 128 and max(s.rq) < 128 else 1)
    if s.n:
        assert got[0] == s.n


def test_query_rows_hit_the_tile_edges():
    for G in GROUPS:
        m = tile_rows(G)
        for D in (64, 256):
            rq, rk = case_lengths("edges", G, D)
            BN = 64 if D > 128 else 128
            assert max(rq) == 127 and {0, 1, m - 1, m, m + 1} <= set(rq) and (2 * m + 1 in rq or 2 * m + 1 > 127)
            assert {0, 1, BN - 1, BN + 1} <= set(rk) and max(rk) == (3000 if G < 64 else 300)
            deltas = [c - r for r, c in zip(rq, rk)]
            assert len(set(deltas)) == len(deltas)
        assert max(case_lengths("full", G, 64)[0]) == 128


@pytest.mark.parametrize("window", [None, (5, 0), (3, 4)])
def test_reversed_heads_permute_the_reference_outputs(window):
    """Reversing the query heads inside every K/V group permutes the float64 reference's O and L the same way."""
    H, G, D = 6, 3, 8
    rq, rk = [3, 0, 5], [4, 6, 2]
    qo, ko = _offsets(rq), _offsets(rk)
    rng = np.random.default_rng(2)
    x = {Op.Q: rng.standard_normal((H, qo[-1], D)), Op.K: rng.standard_normal((H // G, ko[-1], D)),
         Op.V: rng.standard_normal((H // G, ko[-1], D)), Op.dO: np.zeros((H, qo[-1], D))}
    perm = reversed_heads(H, G)
    assert sorted(perm) == list(range(H)) and all(p // G == h // G for h, p in enumerate(perm))
    assert list(perm[:G]) == [2, 1, 0]
    run = ((lambda y: reference(y, G, qo, ko, True)) if window is None else
           (lambda y: band_reference(y, G, qo, ko, *window)))
    base, moved = run(x), run({**x, Op.Q: x[Op.Q][perm]})
    for name in ("O", "L"):
        assert np.array_equal(moved[name], base[name][perm]), name
    assert not np.array_equal(base["O"], base["O"][perm])


@pytest.mark.parametrize("causal,window", [(True, (63, 0)), (False, (40, 20))])
def test_band_poisoned_table_keeps_every_page_a_row_sees(causal, window):
    """Every key that some row of its sequence sees is read through an unchanged page-table entry."""
    rq, rk = [1, 3, 0, 100], [700, 64, 50, 400]
    page = 16
    qo, ko = _offsets(rq), _offsets(rk)
    K = np.random.default_rng(0).standard_normal((1, ko[-1], 4)).astype(np.float32)
    Kp, _, table = build_pool(K, K, ko, page, np.random.default_rng(0))
    poisoned, n = band_poisoned_table(table, rq, rk, page, window, causal, Kp.shape[0])
    assert n > 0
    left, right = window[0], 0 if causal else window[1]
    for s, (Rs, Cs) in enumerate(zip(rq, rk)):
        seen = band_mask(Rs, Cs, left, right).any(axis=0) if Rs else np.zeros(Cs, bool)
        for j in np.flatnonzero(seen):
            assert poisoned[s, j // page] == table[s, j // page], (s, j)


# ------------------------------------------------------------------------------------------------ GPU
def _check_reference(out, ref, qo, mode, prec_L):
    """O within the packed suite's bars; L within 1e-3 plus the rounding of its storage format; rows that see no key
    get L = +inf and O = 0; every other row is finite."""
    T = qo[-1]
    O, L = out["O"][:, :T], out["L"][:, :T]
    rO, rL = ref["O"][:, :T], ref["L"][:, :T]
    empty = np.isposinf(rL)
    assert (np.isposinf(L) == empty).all(), "L = +inf exactly on the rows that see no key"
    assert (O[empty] == 0).all(), "O = 0 on the rows that see no key"
    assert np.isfinite(O[~empty]).all() and np.isfinite(L[~empty]).all()
    _check_within(rO, O, 2e-2 if mode == "bf16" else 5e-3, "O")
    ref_L = np.where(empty, 0.0, rL)
    _check_within(ref_L, np.where(empty, 0.0, L / LOG2E), 1e-3 + storage_error(ref_L * LOG2E, prec_L) / LOG2E, "L")


def _check_raw_L(run, qo, ref):
    """A 16-bit L: +inf is 0x7C00 on the rows that see no key, and rows past the table's end keep 0xFFFF."""
    if run.prec_L == P.FP32:
        return
    raw = run.L.cpu().numpy().view(np.uint16).reshape(run.H, run.T)
    assert (raw[:, qo[-1]:] == 0xFFFF).all(), "16-bit L sentinels"
    assert (raw[:, :qo[-1]][np.isposinf(ref["L"][:, :qo[-1]])] == 0x7C00).all(), "FP16 +inf"


def _poison(run):
    import torch
    run.O.fill_(float("nan"))
    run.L.fill_(float("nan") if run.L.dtype == torch.float32 else -1)


def _same_permuted(moved, base, perm):
    for name in ("O", "L"):
        assert moved[name].tobytes() == np.ascontiguousarray(base[name][perm]).tobytes(), f"reversed heads: {name}"


def _mode(s):
    return "fp16" if s.mode == "reference" else s.mode


def _check_packed(s):
    x, G = s.x, s.G
    runs = []
    for _ in range(2):   # two runs, each after a larger split call (16 ranges) left finite partials in the workspace
        run_packed_split(s.desc, G, x[Op.Q], x[Op.K], x[Op.V], s.qo, s.ko, mfa.SplitKV(16))
        runs.append(run_packed_split(s.desc, G, x[Op.Q], x[Op.K], x[Op.V], s.qo, s.ko, s.split))
    out = runs[0]
    _same(out, runs[1])
    if s.n == 1:
        _same(out, run_packed_forward(s.desc, G, x[Op.Q], x[Op.K], x[Op.V], s.qo, s.ko))
    if s.n and s.D % 8 == 0:
        _same(run_paged_split(s.desc, G, x[Op.Q], s.Kp, s.Vp, s.qo, s.rk, s.table, s.split), out, rows=s.qo[-1])
    perm = reversed_heads(s.H, G)
    _same_permuted(run_packed_split(s.desc, G, x[Op.Q][perm], x[Op.K], x[Op.V], s.qo, s.ko, s.split), out, perm)
    _check_sentinels(out, s.qo)
    _check_reference(out, s.reference(x), s.qo, _mode(s), s.desc.memoryPrecisions[Op.L])


def _check_paged(s):
    x, G = s.x, s.G
    ref = s.reference(x)
    run = SplitPagedRun(s.desc, G, x[Op.Q], s.Kp, s.Vp, s.qo, s.rk, s.table, split=s.split)
    outs = []
    for _ in range(2):   # two runs, each after a larger split call left finite partials in the workspace
        run_paged_split(s.desc, G, x[Op.Q], s.Kp, s.Vp, s.qo, s.rk, s.table, mfa.SplitKV(16))
        _poison(run)
        run.encode()
        outs.append(run.results())
        _check_raw_L(run, s.qo, ref)
    out = outs[0]
    _same(out, outs[1])
    if s.n == 1:
        _same(out, run_paged_plain(s.desc, G, x[Op.Q], s.Kp, s.Vp, s.qo, s.rk, s.table))
    if s.n:
        _same(out, run_packed_split(s.desc, G, x[Op.Q], x[Op.K], x[Op.V], s.qo, s.ko, s.split), rows=s.qo[-1])
    perm = reversed_heads(s.H, G)
    _same_permuted(run_paged_split(s.desc, G, x[Op.Q][perm], s.Kp, s.Vp, s.qo, s.rk, s.table, s.split), out, perm)
    if s.window is not None:
        # pages wholly outside the band of the sequence's rows: a NaN page, or far outside the pool
        Kn, Vn = (np.concatenate([p_, np.full((1,) + p_.shape[1:], np.nan, np.float32)]) for p_ in (s.Kp, s.Vp))
        poisoned, n = band_poisoned_table(s.table, s.rq, s.rk, s.page, s.window, s.causal, s.Kp.shape[0])
        assert n > 0
        _same(out, run_paged_split(s.desc, G, x[Op.Q], Kn, Vn, s.qo, s.rk, poisoned, s.split))
    _check_sentinels(out, s.qo)
    _check_reference(out, ref, s.qo, _mode(s), run.prec_L)


def _scale_sets(s):
    """(k_scale, v_scale, bitwise) per K/V head: NULL scales; or distinct powers of two (V's reversed against K's) and
    distinct scales from each head's absolute maximum, as a serving engine calibrates them (no bitwise identity)."""
    if s.form == "fp8":
        return [(None, None, True)]
    k = (2.0 ** -(2 + np.arange(s.Hkv))).astype(np.float32)
    rng = np.random.default_rng(s.seed)
    # (the head's absolute maximum maps to 400 or less, inside E4M3's 448)
    calibrated = [(np.abs(s.x[op]).max(axis=(1, 2)) / 400 * rng.uniform(1.0, 1.5, s.Hkv)).astype(np.float32)
                  for op in (Op.K, Op.V)]
    return [(k, (2 * k)[::-1].copy(), True), (*calibrated, False)]


def _check_fp8(s):
    G = s.G
    ones = np.ones(s.Hkv, np.float32)
    perm = reversed_heads(s.H, G)
    for k_scale, v_scale, bitwise in _scale_sets(s):
        sk, sv = (ones if a is None else a for a in (k_scale, v_scale))
        Kq, Vq = quantize(s.x[Op.K], sk), quantize(s.x[Op.V], sv)
        Kp, Vp, table = build_pool(Kq, Vq, s.ko, s.page, np.random.default_rng(s.seed))
        x = {**s.x, Op.K: Kq * sk[:, None, None], Op.V: Vq * sv[:, None, None]}
        ref = s.reference(x)
        run = Fp8PagedRun(s.desc, G, x[Op.Q], Kp, Vp, s.qo, s.rk, table, k_scale, v_scale, split=s.split)
        stale = Fp8PagedRun(s.desc, G, x[Op.Q], Kp, Vp, s.qo, s.rk, table, k_scale, v_scale, split=mfa.SplitKV(16))
        outs = []
        for _ in range(2):
            stale.encode()
            _poison(run)
            run.encode()
            outs.append(run.results())
            _check_raw_L(run, s.qo, ref)
        out = outs[0]
        _same(out, outs[1])
        if bitwise:
            Kd, Vd = dequantize(Kp, sk), dequantize(Vp, sv)
            _same(out, run_paged_split(s.desc, G, x[Op.Q], Kd, Vd, s.qo, s.rk, table, s.split))
            if s.n == 1:
                _same(out, run_paged_plain(s.desc, G, x[Op.Q], Kd, Vd, s.qo, s.rk, table))
        moved = Fp8PagedRun(s.desc, G, x[Op.Q][perm], Kp, Vp, s.qo, s.rk, table, k_scale, v_scale, split=s.split)
        moved.encode()
        _same_permuted(moved.results(), out, perm)
        _check_sentinels(out, s.qo)
        _check_reference(out, ref, s.qo, _mode(s), run.prec_L)


def _check_case(*case):
    """Every check of one case, on the GPU (the window, if any, applies to every kernel the runners create)."""
    import contextlib
    from tests.test_window import windowed
    s = Case(*case)
    with windowed(s.window) if s.window else contextlib.nullcontext():
        {"packed": _check_packed, "paged": _check_paged}.get(s.form, _check_fp8)(s)


# Each case runs in a process of its own (see tests/test_paged_fp8_kv.py: the profiler-trace tests of the host API,
# split and packed suites are fragile to GPU work run before them in the same session).  A fresh interpreter spends
# about 7 s importing torch against about 1 s of checks, so the processes are forked from a multiprocessing fork
# server that imported torch once and never touches the GPU; each child imports this module, creates its own CUDA
# context and exits after its case.  The child sends the records of its checks as JSON, and they join this session's
# records.
_FORK_SERVER = None


def _child(case, test_name, conn):
    import traceback
    from tests import attention_harness
    os.environ["PYTEST_CURRENT_TEST"] = test_name   # (the fork server's environment is that of the first case)
    try:
        _check_case(*case)
        conn.send(("passed", json.dumps(attention_harness.RECORDS)))
    except BaseException:
        conn.send(("failed", traceback.format_exc()))
    conn.close()


def _isolated(case):
    import multiprocessing
    from tests import attention_harness
    global _FORK_SERVER
    if _FORK_SERVER is None:
        _FORK_SERVER = multiprocessing.get_context("forkserver")
        _FORK_SERVER.set_forkserver_preload(["torch"])
    receive, send = _FORK_SERVER.Pipe(duplex=False)
    child = _FORK_SERVER.Process(target=_child, args=(case, os.environ.get("PYTEST_CURRENT_TEST", ""), send))
    child.start()
    send.close()
    status, payload = "timed out", "the case did not finish within 900 s"
    if receive.poll(900):
        try:
            status, payload = receive.recv()
        except EOFError:   # (the child exited without reporting)
            child.join()
            status, payload = "died", f"the child process exited with code {child.exitcode}"
    child.join(60 if status != "timed out" else 0)
    if child.is_alive():
        child.kill()
        child.join()
    assert status == "passed", payload
    attention_harness.RECORDS.extend(json.loads(payload))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_grouped_decode(case):
    _isolated(case)
