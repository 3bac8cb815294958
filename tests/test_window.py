"""Sliding-window attention (AttentionKernel(kd, window=(left, right)), AttentionKernel.cached(..., window=)).

With delta = C - R (Cs - Rs per sequence in packed and paged calls), query row i sees key j iff
i + delta - left <= j <= i + delta + right, and -1 leaves a side unbounded.  A row that sees no key gets O = 0,
L = +inf, D = 0, dQ = 0; a key that no row sees gets dK = dV = 0.

The GPU cases reuse the grouped, packed and paged suites' runners unchanged: `windowed(window)` makes the kernels they
create windowed ones.  Each case is checked against a float64 band reference with those suites' tolerances, and a
second run must be bitwise identical.  Bitwise identities pin the band kernels to the existing ones where they must
agree, and the paged cases show that out-of-window pages are never read."""
import contextlib
import ctypes
import os
import re

import numpy as np
import pytest

import mfa_b200 as mfa
from tests.causal_oracle import attention_f64
from tests.test_varlen import LOG2E, _check_against_reference, _constants, _offsets
from tests.test_varlen import _descriptor as varlen_descriptor

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
INT32_MAX = 2**31 - 1


# ------------------------------------------------------------------------------------------------ the reference
def band_mask(R, C, left, right):
    """[R, C] boolean: True where query row i sees key j."""
    d = np.arange(C)[None, :] - np.arange(R)[:, None] - (C - R)   # key - (row + delta)
    mask = np.ones((R, C), bool)
    if right >= 0:
        mask &= d <= right
    if left >= 0:
        mask &= -d <= left
    return mask


def band_attention_f64(Q, K, V, dO, left, right):
    """attention_f64 under the band: O, L (natural log), D, dQ, dK, dV in float64."""
    Q, K, V, dO = (np.asarray(x, np.float64) for x in (Q, K, V, dO))
    R, D = Q.shape
    C = K.shape[0]
    scale = 1.0 / np.sqrt(D)
    mask = band_mask(R, C, left, right)
    S = np.where(mask, (Q @ K.T) * scale, -np.inf)
    m = S.max(axis=1, keepdims=True) if C else np.full((R, 1), -np.inf)
    empty = ~np.isfinite(m[:, 0])
    m = np.where(np.isfinite(m), m, 0.0)
    E = np.exp(S - m)
    lsum = E.sum(axis=1, keepdims=True)
    Pm = E / np.where(lsum > 0, lsum, 1.0)
    O = Pm @ V
    Dt = (dO * O).sum(axis=1)
    dS = Pm * ((dO @ V.T) - Dt[:, None]) * scale
    return {"O": O, "L": np.where(empty, np.inf, (m + np.log(np.where(lsum > 0, lsum, 1.0)))[:, 0]), "D": Dt,
            "dQ": dS @ K, "dK": dS.T @ Q, "dV": Pm.T @ dO}


def band_reference(inputs, G, qo, ko, left, right):
    """band_attention_f64 of every (sequence, head) in the packed layout of tests/test_varlen.reference."""
    Q, K, V, dO = (np.asarray(inputs[op], np.float64) for op in (Op.Q, Op.K, Op.V, Op.dO))
    H = Q.shape[0]
    out = {"O": np.zeros_like(Q), "dQ": np.zeros_like(Q), "L": np.zeros(Q.shape[:2]), "D": np.zeros(Q.shape[:2]),
           "dK": np.zeros_like(K), "dV": np.zeros_like(V)}
    for s in range(len(qo) - 1):
        q, k = slice(qo[s], qo[s + 1]), slice(ko[s], ko[s + 1])
        for h in range(H):
            r = band_attention_f64(Q[h, q], K[h // G, k], V[h // G, k], dO[h, q], left, right)
            for name in ("O", "dQ", "L", "D"):
                out[name][h, q] = r[name]
            out["dK"][h // G, k] += r["dK"]
            out["dV"][h // G, k] += r["dV"]
    return out


@pytest.mark.parametrize("R,C,left,right", [(37, 53, 5, 0), (53, 37, 3, 2), (40, 40, 0, 5), (30, 70, 300, -1),
                                            (64, 64, -1, 7), (20, 9, 1, 0)])
def test_band_reference_matches_torch_sdpa_with_an_explicit_mask(R, C, left, right):
    import torch
    rng = np.random.default_rng(R * C + left)
    D = 16
    Q, K, V, dO = (rng.standard_normal((n, D)) for n in (R, C, C, R))
    ref = band_attention_f64(Q, K, V, dO, left, right)
    mask = band_mask(R, C, left, right)
    seen = mask.any(axis=1)   # rows that see no key are NaN in torch; the library's rule gives them O = 0
    tq, tk, tv = (torch.tensor(a, requires_grad=True) for a in (Q, K, V))
    O = torch.nn.functional.scaled_dot_product_attention(tq[None], tk[None], tv[None], attn_mask=torch.tensor(mask))[0]
    O = torch.where(torch.tensor(seen)[:, None], O, torch.zeros_like(O))
    (O * torch.tensor(dO)).sum().backward()
    for name, got in (("O", O.detach()), ("dQ", tq.grad), ("dK", tk.grad), ("dV", tv.grad)):
        assert np.abs(np.nan_to_num(got.numpy()) - ref[name]).max() <= 1e-10, name
    assert np.isposinf(ref["L"][~seen]).all() and np.isfinite(ref["L"][seen]).all()
    assert (ref["dK"][~mask.any(axis=0)] == 0).all() and (ref["dV"][~mask.any(axis=0)] == 0).all()


@pytest.mark.parametrize("R,C", [(40, 40), (25, 60), (60, 25)])
def test_unbounded_band_is_the_causal_oracle(R, C):
    rng = np.random.default_rng(R + C)
    Q, K, V, dO = (rng.standard_normal((n, 8)) for n in (R, C, C, R))
    for causal, window in ((False, (-1, -1)), (True, (-1, 0)), (True, (INT32_MAX, 0)), (False, (INT32_MAX, INT32_MAX))):
        ref, band = attention_f64(Q, K, V, dO, causal=causal), band_attention_f64(Q, K, V, dO, *window)
        for name in ref:
            assert np.allclose(band[name], ref[name], rtol=1e-12, atol=1e-12, equal_nan=False), (causal, name)


# ------------------------------------------------------------------------------------------------ CPU: the API
def _kd(mode="bf16", causal=False, t=KT.forward, D=128, R=4096, C=4096):
    return varlen_descriptor(R, C, D, mode, 1, causal).kernelDescriptor(t)


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_invalid_windows_are_rejected(mode):
    bad = [((-2, 0), False, "left -2 is below -1"), ((0, -5), False, "right -5 is below -1"),
           ((3, 1), True, "right 1 on a causal kernel")]
    for t in KT:
        for window, causal, message in bad:
            with pytest.raises(mfa.MFAError) as e:
                mfa.AttentionKernel(_kd(mode, causal, t), window=window)
            assert e.value.status == -2 and "Window" in e.value.message and message in e.value.message, e.value.message
            desc = varlen_descriptor(128, 128, 64, mode, 1, causal)
            with pytest.raises(mfa.MFAError) as e:
                mfa.AttentionKernel.cached(desc, t, window=window)
            assert e.value.status == -2 and message in e.value.message, e.value.message
    # values the C struct cannot hold are not wrapped into it
    for window in ((2**32 - 1, 0), (0, 2**31), (-2**31 - 1, 0)):
        with pytest.raises(mfa.MFAError) as e:
            mfa.AttentionKernel(_kd(mode), window=window)
        assert e.value.status == -2 and "is outside [-1, 2147483647]" in e.value.message, e.value.message
        with pytest.raises(mfa.MFAError):
            mfa.AttentionKernel.cached(varlen_descriptor(128, 128, 64, mode, 1, False), KT.forward, window=window)
    # NULL windows through the C entry points
    kd, desc, out = _kd(mode), varlen_descriptor(128, 128, 64, mode, 1, False)._c(), ctypes.c_void_p()
    for status in (mfa._lib.mfa_attention_kernel_create_windowed(ctypes.byref(kd._c), None, ctypes.byref(out)),
                   mfa._lib.mfa_attention_kernel_cache_fetch_windowed(ctypes.byref(desc), 0, None, ctypes.byref(out))):
        assert status == -2 and "NULL window" in mfa._lib.mfa_last_error().decode()
    # every value in [-1, INT32_MAX] is accepted; a causal kernel takes right 0 or -1
    for window in ((-1, -1), (0, 0), (INT32_MAX, INT32_MAX), (0, INT32_MAX)):
        mfa.AttentionKernel(_kd(mode), window=window)
    for window in ((-1, 0), (0, -1), (INT32_MAX, 0)):
        mfa.AttentionKernel(_kd(mode, True), window=window)


def test_source_names_and_cache_keys():
    k = mfa.AttentionKernel(_kd("bf16", True), window=(4095, 0))
    assert k.sourceName() == "attention_forward_tcgen05<D=128>_causal_window<4095,0>"
    k = mfa.AttentionKernel(_kd("fp32", False, KT.backwardKeyValue, D=64), window=(-1, 7))
    assert k.sourceName() == "attention_backward_key_value_simt_fp32<D=64>_window<-1,7>"
    assert mfa.AttentionKernel(_kd("bf16")).sourceName() == "attention_forward_tcgen05<D=128>"
    assert "sliding window" in mfa.version() and " 0.5 " in mfa.version()
    desc = varlen_descriptor(333, 333, 64, "bf16", 1, True)
    for t in KT:
        a = mfa.AttentionKernel.cached(desc, t, window=(100, 0))
        assert mfa.AttentionKernel.cached(desc, t, window=(100, 0))._handle.value == a._handle.value
        b = mfa.AttentionKernel.cached(desc, t, window=(101, 0))
        plain = mfa.AttentionKernel.cached(desc, t)
        assert len({a._handle.value, b._handle.value, plain._handle.value}) == 3
        assert mfa.AttentionKernel.cached(desc, t)._handle.value == plain._handle.value
        assert b.sourceName().endswith("_causal_window<101,0>") and "window" not in plain.sourceName()


def test_launch_counts_of_windowed_calls():
    """132 SMs without a device.  A decode-shaped windowed forward splits over the band's blocks (34 of 128 keys for a
    (4095, 0) window: 2 ranges of 17), and launches one kernel when splitting is off; packed and paged calls never
    split."""
    def count(window, policy=None, t=KT.forward, R=1, C=32768, D=128, mode="bf16"):
        kd = _kd(mode, True, t, D)
        if policy is not None:
            kd.splitPolicy = policy
        return mfa.AttentionKernel(kd, window=window).launchCount(_constants(R, C, 1, 1))
    assert count((4095, 0)) == 2
    assert count((4095, 0), (0, 1)) == 1
    assert count((4095, 0), (8, 4)) == 2           # 34 blocks: 2 ranges of 17 (4 does not divide 34)
    assert count((1, 0)) == 1                      # two blocks at most: too few to split
    plain = mfa.AttentionKernel(_kd("bf16", True)).launchCount(_constants(1, 32768, 1, 1))
    assert count((-1, 0)) == plain                 # the unbounded window plans as the causal kernel
    for t in (KT.backwardQuery, KT.backwardKeyValue):
        assert count((4095, 0), None, t, R=64, C=32768) >= 1
        assert count((4095, 0), (0, 1), t, R=64, C=32768) == 1
    table = mfa.SequenceTable(3, 100, 3000, 16, 16)
    k = mfa.AttentionKernel(_kd("bf16", True), window=(63, 0))
    assert k.launchCount(_constants(300, 9000, 1, 1), table) == 1
    paged = mfa.PagedKV(2, 10, 16, 16, 16, 4, 16)
    assert k.launchCount(_constants(16, 1024, 1, 1), paged=paged) == 1


def test_cpp_host_mirror_with_a_window(tmp_path):
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
  d.matrixDimensions = MatrixDimensions{1, 32768, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  d.causal = true;
  mfa_function_constants_t constants;
  d.setFunctionConstants(constants);
  AttentionKernel own(d.kernelDescriptor(AttentionKernelType::forward), AttentionWindow{4095, 0});
  AttentionKernel cached(d, AttentionKernelType::forward, AttentionWindow{4095, 0});
  std::printf("%s %u %zu\n", cached.sourceName().c_str(), own.launchCount(constants), sizeof(AttentionWindow));
  try {
    AttentionKernel bad(d.kernelDescriptor(AttentionKernelType::forward), AttentionWindow{4095, 3});
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
    assert out == ["attention_forward_tcgen05<D=128>_causal_window<4095,0>", "2", "8", "rejected"], out


def test_ptxas_band_tensor_core_kernels_have_no_spills_and_no_stack_frame():
    from tests.test_forward_pipeline import _ptxas_report
    report, text = _ptxas_report()
    kernels = {name: r for name, r in report.items() if re.search(r"band_\w+_wgmma", name)}
    # forward: 3 head-dimension chunk counts x bf16 / fp16 x (fixed, packed, paged); dQ and dK/dV: 3 x (bf16, fp16,
    # fp16 with BF16 dO) x (fixed, packed)
    assert len(kernels) == 3 * 2 * 3 + 2 * 3 * 3 * 2, sorted(kernels)
    for name, r in kernels.items():
        assert not re.search(r"attention_\w+_wgmma", name) and "paged_forward_wgmma" not in name, name
        assert r == (0, 0, 0), (name, r)
        assert not re.search(r"C7510.*" + re.escape(name), text), name


# ------------------------------------------------------------------------------------------------ GPU
@contextlib.contextmanager
def windowed(window):
    """Within the block, every AttentionKernel(kd) the suites' runners create is AttentionKernel(kd, window=window)."""
    plain = mfa.AttentionKernel

    class Windowed(plain):
        def __init__(self, descriptor, window_=None):
            super().__init__(descriptor, window=window)

    mfa.AttentionKernel = Windowed
    try:
        yield
    finally:
        mfa.AttentionKernel = plain


def _split(policy):
    def edit(kd):
        if policy is not None:
            kd.splitPolicy = policy
    return edit


def _fixed(R, C, D, mode, H, G, causal, window, policy=None, transpose=(False,) * 4, seed=0):
    """A fixed-length windowed forward + backward against the band reference; returns the raw outputs."""
    from tests.test_kv_group import _descriptor, _inputs, run
    desc = _descriptor(R, C, D, mode, batch=H, causal=causal, transpose=transpose)
    x = _inputs(desc, G, seed)
    with windowed(window):
        out = run(desc, G, x, edit=_split(policy), raw=True)
        again = run(desc, G, x, edit=_split(policy), raw=True)
    for name in out:
        assert out[name].tobytes() == again[name].tobytes(), f"second run differs in {name}"
    left, right = window
    ref = band_reference(x, G, [0, R], [0, C], left, 0 if causal else right)
    _check_against_reference(out, ref, [0, R], [0, C], "fp16" if mode == "reference" else mode, G, D)
    return out


LEFTS = [0, 1, 63, 64, 127, 128, 129, 777, INT32_MAX]
FIXED = [  # (R, C, D, mode, H, G, causal, window, split policy)
    *[(300, 300, 128, "bf16", 4, 4, True, (left, 0), None) for left in LEFTS],
    (200, 520, 64, "fp16", 4, 1, True, (129, 0), None), (520, 200, 64, "bf16", 4, 4, True, (63, -1), None),
    (256, 256, 256, "bf16", 2, 1, True, (128, 0), (0, 1)), (384, 384, 128, "reference", 4, 4, False, (128, 128), None),
    (300, 300, 64, "bf16", 4, 1, False, (0, 5), None), (200, 700, 128, "fp16", 4, 4, False, (300, -1), None),
    (700, 200, 64, "reference", 4, 1, False, (5, 0), None), (130, 130, 256, "fp16", 2, 1, False, (64, 64), (0, 1)),
    (64, 4096, 128, "bf16", 4, 4, True, (777, 0), (2, 8)), (1, 8192, 64, "bf16", 4, 1, True, (1023, 0), (2, 8)),
    (64, 4096, 128, "reference", 4, 4, False, (300, 200), (2, 8)), (200, 300, 60, "bf16", 4, 1, True, (64, 0), None),
    (300, 300, 60, "fp16", 4, 4, False, (128, 128), None),
    (150, 150, 32, "fp32", 4, 4, True, (63, 0), None), (90, 200, 72, "fp32", 4, 1, False, (0, 5), None),
    (200, 90, 320, "fp32", 2, 1, False, (300, -1), None), (129, 129, 64, "fp32", 4, 4, False, (INT32_MAX, 1), None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode,H,G,causal,window,policy", FIXED)
def test_windowed_fixed_calls_match_the_band_reference(R, C, D, mode, H, G, causal, window, policy):
    _fixed(R, C, D, mode, H, G, causal, window, policy, seed=R + C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,transpose", [("bf16", 128, (True,) * 4), ("fp16", 64, (False, True, True, False)),
                                              ("fp32", 64, (True, False, True, True))])
def test_windowed_transposed_operands(mode, D, transpose):
    _fixed(192, 256, D, mode, 2, 1, True, (100, 0), None, transpose)
    _fixed(256, 192, D, mode, 2, 2, False, (30, 70), None, transpose)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D", [("bf16", 128), ("fp16", 64), ("reference", 256), ("fp32", 64)])
def test_unbounded_bands_equal_the_existing_kernels_bitwise(mode, D):
    """(-1, -1) on an unmasked kernel and (-1, 0) on a causal one, splitting off: the band kernels run the same
    instructions on every block they share with the existing kernels."""
    from tests.test_kv_group import _descriptor, _inputs, run
    for R, C, causal, window in ((300, 300, False, (-1, -1)), (200, 333, True, (-1, 0)), (333, 200, True, (-1, 0))):
        desc = _descriptor(R, C, D, mode, batch=4, causal=causal)
        x = _inputs(desc, 2, 5)
        plain = run(desc, 2, x, edit=_split((0, 1)), raw=True)
        with windowed(window):
            band = run(desc, 2, x, edit=_split((0, 1)), raw=True)
        for name in plain:
            assert plain[name].tobytes() == band[name].tobytes(), (R, C, causal, name)


PACKED = [  # (mode, D, causal, G, window, query lengths, key lengths)
    ("bf16", 128, True, 4, (63, 0), [70, 1, 130, 200, 0], [90, 64, 130, 100, 20]),
    ("fp16", 64, False, 1, (20, 40), [64, 65, 3], [200, 65, 0]),
    ("reference", 256, True, 4, (128, -1), [129, 1, 300], [129, 500, 100]),
    ("fp32", 64, True, 4, (5, 0), [70, 1, 130], [90, 64, 100]),
    ("fp32", 96, False, 1, (-1, 3), [33, 80], [80, 33]),
    ("fp32", 64, False, 1, (20, 40), [64, 65, 3], [200, 65, 0]),    # Cs = 0 under a band that reaches the diagonal
    ("fp32", 64, False, 4, (-1, -1), [10, 0, 7], [0, 5, 9]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,G,window,rq,rk", PACKED)
def test_windowed_packed_calls(mode, D, causal, G, window, rq, rk):
    """The band reference per sequence, untouched sentinels, a bitwise second run, and with a tensor-core kernel each
    sequence bitwise equal to a windowed fixed-length call on it alone."""
    from tests.test_varlen import _check_sentinels, _inputs, _per_sequence_bitwise, run_packed
    qo, ko = _offsets(rq), _offsets(rk)
    H = 4
    T, Tk = qo[-1] + 7, ko[-1] + 5
    desc = varlen_descriptor(T, Tk, D, mode, H, causal)
    x = _inputs(desc, G, T, Tk, seed=D + G)
    with windowed(window):
        out = run_packed(desc, G, x, qo, ko)
        again = run_packed(desc, G, x, qo, ko)
        for name in out:
            assert out[name].tobytes() == again[name].tobytes(), name
        _check_sentinels(out, qo, ko)
        if mode != "fp32":
            _per_sequence_bitwise(desc, G, x, out, qo, ko)
    left, right = window
    ref = band_reference(x, G, qo, ko, left, 0 if causal else right)
    _check_against_reference(out, ref, qo, ko, "fp16" if mode == "reference" else mode, G, D)


def _paged_case(mode, D, causal, G, window, rq, rk, page_size, seed, fill=None):
    from tests.test_paged_kv import build_pool
    from tests.test_varlen import _inputs
    qo, ko = _offsets(rq), _offsets(rk)
    H = 4
    T, Tk = qo[-1] + 9, ko[-1] + 5
    desc = varlen_descriptor(T, Tk, D, mode, H, causal)
    x = _inputs(desc, G, T, Tk, seed)
    Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, page_size, np.random.default_rng(seed), fill=fill)
    return desc, x, qo, ko, Kp, Vp, table


PAGED = [  # (mode, D, causal, G, window, page size, query lengths, key lengths)
    ("bf16", 128, True, 4, (100, 0), 16, [1, 1, 1, 60], [1, 100, 333, 150]),
    ("fp16", 64, True, 1, (63, 0), 32, [1, 1, 70], [700, 64, 300]),
    ("reference", 256, False, 4, (40, 20), 64, [3, 100, 1], [300, 90, 1000]),
    ("bf16", 64, True, 1, (0, 0), 256, [1, 5, 200], [1000, 50, 100]),
    ("fp32", 64, True, 4, (100, 0), 16, [1, 1, 60], [333, 100, 150]),
    ("fp32", 72, False, 1, (30, 5), 32, [1, 100], [500, 90]),
    ("fp32", 64, False, 1, (0, 3), 16, [5, 3, 7], [100, 0, 30]),      # Cs = 0
    ("bf16", 64, False, 4, (0, 3), 16, [5, 3, 7], [100, 0, 30]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,G,window,page_size,rq,rk", PAGED)
def test_windowed_paged_forward(mode, D, causal, G, window, page_size, rq, rk):
    """Bitwise equal to the windowed packed forward on the same keys, and to itself with every page outside the band
    of the sequence's rows replaced by a NaN page: those pages, and their page-table entries, are never read."""
    from tests.test_paged_kv import _check_reference, _check_sentinels, run_packed_forward, run_paged_forward
    desc, x, qo, ko, Kp, Vp, table = _paged_case(mode, D, causal, G, window, rq, rk, page_size, seed=D + page_size)
    Q = x[Op.Q]
    left, right = window[0], 0 if causal else window[1]
    with windowed(window):
        packed = run_packed_forward(desc, G, Q, x[Op.K], x[Op.V], qo, ko)
        paged = run_paged_forward(desc, G, Q, Kp, Vp, qo, rk, table)
        again = run_paged_forward(desc, G, Q, Kp, Vp, qo, rk, table)
        # every page-table entry whose page lies wholly outside the band of all of its sequence's rows points at a
        # NaN page (appended to the pools), or at a page id far outside the pool
        nan_page = Kp.shape[0]
        Kn, Vn = (np.concatenate([pool, np.full((1,) + pool.shape[1:], np.nan, np.float32)]) for pool in (Kp, Vp))
        poisoned, n = table.copy(), 0
        for s, (Rs, Cs) in enumerate(zip(rq, rk)):
            delta = Cs - Rs
            lo = delta - left if left >= 0 else -np.inf         # the lowest key any row sees
            hi = Rs - 1 + delta + right if right >= 0 else np.inf
            for j in range(-(-Cs // page_size)):
                if (j + 1) * page_size <= lo or j * page_size > hi:
                    poisoned[s, j] = nan_page if n % 2 == 0 else 2**31 - 1
                    n += 1
        if page_size <= 64:
            assert n > 0   # (the cases are chosen so that some pages fall outside the window)
        skipped = run_paged_forward(desc, G, Q, Kn, Vn, qo, rk, poisoned)
    for name in ("O", "L"):
        assert paged[name].tobytes() == again[name].tobytes(), name
        assert paged[name][:, :qo[-1]].tobytes() == packed[name][:, :qo[-1]].tobytes(), name
        assert skipped[name].tobytes() == paged[name].tobytes(), name
    _check_sentinels(paged, qo)
    ref = band_reference({Op.Q: Q, Op.K: x[Op.K], Op.V: x[Op.V], Op.dO: np.zeros_like(Q)}, G, qo, ko, left, right)
    _check_reference(paged, ref, qo, "fp16" if mode == "reference" else mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("causal,window", [(False, (10, -1)), (False, (-1, -1)), (True, (-1, 0)), (False, (3, 2))])
def test_windowed_paged_forward_with_a_page_table_of_two_billion_keys(mode, causal, window):
    """page_stride x P = 2^31: an unbounded side resolves to INT32_MAX, and the band's edges (delta + right, delta -
    left) leave int32.  The output equals, bit for bit, the same call with a page table just long enough."""
    from tests.test_paged_kv import _check_reference, run_paged_forward
    P_ = 256
    desc, x, qo, ko, Kp, Vp, table = _paged_case(mode, 64, causal, 2, window, [1, 40], [700, 300], P_, seed=41)
    long_table = np.zeros((table.shape[0], 2**31 // P_), np.int64)
    long_table[:, :table.shape[1]] = table
    with windowed(window):
        short = run_paged_forward(desc, 2, x[Op.Q], Kp, Vp, qo, [700, 300], table)
        long = run_paged_forward(desc, 2, x[Op.Q], Kp, Vp, qo, [700, 300], long_table)
    for name in ("O", "L"):
        assert long[name].tobytes() == short[name].tobytes(), name
    left, right = window[0], 0 if causal else window[1]
    ref = band_reference({Op.Q: x[Op.Q], Op.K: x[Op.K], Op.V: x[Op.V], Op.dO: np.zeros_like(x[Op.Q])}, 2, qo, ko,
                         left, right)
    _check_reference(long, ref, qo, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_windowed_paged_decode_replays_in_a_cuda_graph_as_the_cache_grows(mode):
    """A captured windowed decode step replayed while the cache grows past the window: each replay equals a fresh call,
    and matches the band reference."""
    import torch
    from tests.test_paged_kv import PagedRun, _check_reference, gather
    window, P_, W = (63, 0), 16, 64
    rq, rk = [1, 1], [40, 90]
    desc, x, qo, ko, Kp, Vp, table = _paged_case(mode, 64, True, 2, window, rq, [300, 300], P_, seed=3)
    with windowed(window):
        run = PagedRun(desc, 2, x[Op.Q], Kp, Vp, qo, rk, table)
        run.encode()
        torch.cuda.synchronize()
        stream = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            run.encode(stream.cuda_stream)
        for step in range(0, 3 * W, 37):
            lengths = [c + step for c in rk]
            run.lengths.copy_(torch.tensor(lengths, dtype=torch.int32))
            run.O.fill_(float("nan"))
            g.replay()
            replayed = run.results()
            fresh = PagedRun(desc, 2, x[Op.Q], Kp, Vp, qo, lengths, table)
            fresh.encode()
            expected = fresh.results()
            for name in ("O", "L"):
                assert replayed[name].tobytes() == expected[name].tobytes(), (step, name)
            Ks, Vs = [], []
            for s, c in enumerate(lengths):
                Ks.append(gather(Kp, table[s:s + 1], [c], P_))
                Vs.append(gather(Vp, table[s:s + 1], [c], P_))
            ko_now = _offsets(lengths)
            ref = band_reference({Op.Q: x[Op.Q], Op.K: np.concatenate(Ks, axis=1), Op.V: np.concatenate(Vs, axis=1),
                                  Op.dO: np.zeros_like(x[Op.Q])}, 2, qo, ko_now, 63, 0)
            _check_reference(replayed, ref, qo, mode)
