"""Grouped-query attention (FunctionConstantValues.kvGroup = G): G query problems share one K/V problem.

Query problem b (Q, O, L, D, dO, dQ) reads K/V problem b // G; K, V, dK and dV hold batch // G problems, and dK / dV
are the sums over the G query problems of a group.  With G = 1 (or 0) this is the ungrouped batch.

The reference is tests/causal_oracle.attention_f64 per query head with the K/V of its group, dK and dV summed over the
group; on the CPU it is pinned against PyTorch's scaled_dot_product_attention(enable_gqa=True).  On the GPU, forward and
dQ must be bitwise identical to the same call on K/V expanded with repeat_interleave (same plan, same arithmetic), dK /
dV must equal the sum of the expanded call's per-head dK / dV up to FP32 reordering, and both must meet the backward
suites' tolerances against the float64 reference.

The launch-count check traces kernels with torch.profiler in a child process, and the module sorts after
tests/test_host_api.py: the profiler's state is process-wide, and the trace windows of tests/test_causal.py and
tests/test_host_api.py (whose windows open with the library's own kernel, which a trace can drop) keep the history of
GPU work they have without this module."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import mfa_b200 as mfa
import oracle
from tests.causal_oracle import attention_f64, causal_mask

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG2E = 1.44269504089
GOLDEN = os.path.join(ROOT, "tests", "golden", "gqa_default_outputs.json")


def _descriptor(R, C, D, mode="bf16", batch=1, causal=False, transpose=(False,) * 4, lowMid=False):
    """mode: "bf16" / "fp16" (all operands of that type), "reference" (FP16 Q/K/V, BF16 dO) or "fp32" (SIMT family).
    lowMid: L stored as FP16 and D as BF16 (lowPrecisionIntermediates)."""
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = mode != "fp32"
    desc.lowPrecisionIntermediates = lowMid
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = tuple(transpose)
    desc.batchCount = batch
    desc.causal = causal
    if mode in ("bf16", "fp16"):
        desc.inputPrecisionOverride = P.BF16 if mode == "bf16" else P.FP16
    return desc


def _inputs(desc, G, seed):
    """Seeded Q, dO [batch, R, D] and K, V [batch / G, C, D], rounded to the operands' memory precisions."""
    R, C, D = desc.matrixDimensions
    B = desc.batchCount
    rng = np.random.default_rng(seed)
    x = {Op.Q: rng.standard_normal((B, R, D)), Op.K: rng.standard_normal((B // G, C, D)),
         Op.V: rng.standard_normal((B // G, C, D)), Op.dO: rng.standard_normal((B, R, D))}
    prec = desc.memoryPrecisions
    return {op: oracle.roundtrip(a.astype(np.float32), int(prec[op])) for op, a in x.items()}


def reference(inputs, G, causal):
    """float64: per query head b, attention_f64 with the K/V of head b // G; dK and dV summed over each group."""
    Q, K, V, dO = (inputs[op] for op in (Op.Q, Op.K, Op.V, Op.dO))
    heads = [attention_f64(Q[b], K[b // G], V[b // G], dO[b], causal=causal) for b in range(Q.shape[0])]
    out = {name: np.stack([h[name] for h in heads]) for name in ("O", "L", "D", "dQ")}
    for name in ("dK", "dV"):
        out[name] = np.stack([sum(heads[b][name] for b in range(g * G, (g + 1) * G)) for g in range(K.shape[0])])
    return out


def expand(inputs, G):
    """The workaround grouped K/V replaces: K and V repeated per query head (torch.repeat_interleave(K, G, dim=0))."""
    return {op: np.repeat(a, G, axis=0) if op in (Op.K, Op.V) else a for op, a in inputs.items()}


# ------------------------------------------------------------------------------------------------ CPU: the reference
@pytest.mark.parametrize("B,Hq,Hkv,R,C,D,causal", [(2, 4, 2, 24, 24, 16, False), (1, 6, 2, 20, 37, 8, True),
                                                   (2, 3, 1, 17, 17, 12, True), (1, 8, 8, 9, 15, 4, False)])
def test_reference_matches_torch_sdpa_enable_gqa(B, Hq, Hkv, R, C, D, causal):
    import torch
    G = Hq // Hkv
    rng = np.random.default_rng(R + C + D)
    q, do = (rng.standard_normal((B, Hq, R, D)) for _ in range(2))
    k, v = (rng.standard_normal((B, Hkv, C, D)) for _ in range(2))
    inputs = {Op.Q: q.reshape(B * Hq, R, D), Op.K: k.reshape(B * Hkv, C, D), Op.V: v.reshape(B * Hkv, C, D),
              Op.dO: do.reshape(B * Hq, R, D)}
    ref = reference(inputs, G, causal)
    tq, tk, tv = (torch.tensor(a, requires_grad=True) for a in (q, k, v))
    mask = torch.tensor(causal_mask(R, C)) if causal else None   # bottom-right aligned; R <= C: no row is empty
    O = torch.nn.functional.scaled_dot_product_attention(tq, tk, tv, attn_mask=mask, enable_gqa=True)
    (O * torch.tensor(do)).sum().backward()
    for name, got in (("O", O.detach()), ("dQ", tq.grad), ("dK", tk.grad), ("dV", tv.grad)):
        got = got.numpy().reshape(ref[name].shape)
        assert np.abs(got - ref[name]).max() <= 1e-10, name


def test_reference_with_one_head_per_group_is_per_head_attention():
    rng = np.random.default_rng(3)
    inputs = {op: rng.standard_normal((3, 19, 8)) for op in (Op.Q, Op.K, Op.V, Op.dO)}
    ref = reference(inputs, 1, True)
    for b in range(3):
        single = attention_f64(*(inputs[op][b] for op in (Op.Q, Op.K, Op.V, Op.dO)), causal=True)
        for name in ("O", "L", "D", "dQ", "dK", "dV"):
            assert np.array_equal(ref[name][b], single[name]), name


# ------------------------------------------------------------------------------------------------ CPU: the API
def _constants(desc, G):
    c = mfa.FunctionConstantValues()
    desc.setFunctionConstants(c)
    assert c.kvGroup == 0, "setFunctionConstants describes no grouping"
    c.kvGroup = G
    return c


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_invalid_groups_are_rejected(mode):
    desc = _descriptor(128, 128, 64, mode, batch=12)
    for t in KT:
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(t))
        for G in (5, 8, 24, 16385):    # batch % G != 0, and G beyond one launch slice
            c = _constants(desc, G)
            for call in (kernel.gridSize, kernel.launchCount):
                with pytest.raises(mfa.MFAError) as e:
                    call(c)
                assert e.value.status == -2
                assert "kv_group" in e.value.message
    big = _descriptor(8, 8, 64, mode, batch=2 * 16385)
    with pytest.raises(mfa.MFAError) as e:
        mfa.AttentionKernel(big.kernelDescriptor(KT.forward)).launchCount(_constants(big, 16385))
    assert "exceeds 16384" in e.value.message


def test_grid_size_and_launch_count_with_groups():
    """dK/dV CTAs own K/V tiles: its grid has batch / G rows, and that CTA count drives the split and dO-conversion
    choices (132 SMs without a device).  Forward and dQ grids do not change."""
    R, C, D, B = 2048, 1024, 128, 32
    for mode in ("bf16", "reference"):
        desc = _descriptor(R, C, D, mode, batch=B)
        kernels = {t: mfa.AttentionKernel(desc.kernelDescriptor(t)) for t in KT}
        par = {t: kernels[t].blockDimensions[0] for t in KT}
        for G in (0, 1, 2, 16, 32):
            c = _constants(desc, G)
            g = max(G, 1)
            assert kernels[KT.forward].gridSize(c) == -(-R // par[KT.forward]) * B
            assert kernels[KT.backwardQuery].gridSize(c) == -(-R // par[KT.backwardQuery]) * B
            assert kernels[KT.backwardKeyValue].gridSize(c) == -(-C // par[KT.backwardKeyValue]) * (B // g)
            ungrouped = _constants(desc, 1)
            for t in (KT.forward, KT.backwardQuery):
                assert kernels[t].launchCount(c) == kernels[t].launchCount(ungrouped)
        kv = kernels[KT.backwardKeyValue]
        # 8 tiles x 32 heads: one full grid, not split; 8 tiles x 2 or 1 K/V heads: split, + sum_splits
        if mode == "bf16":
            assert [kv.launchCount(_constants(desc, G)) for G in (1, 2, 16, 32)] == [1, 1, 2, 2]
        else:   # BF16 dO beside FP16 Q/K/V: converted in a pass of its own on the full grid, on chip on the small one
            assert [kv.launchCount(_constants(desc, G)) for G in (1, 16, 32)] == [2, 2, 2]
            small = _descriptor(128, 1024, 128, mode, batch=B)
            assert mfa.AttentionKernel(small.kernelDescriptor(KT.backwardKeyValue)).launchCount(_constants(small, 16)) == 1


def test_launch_count_slices_whole_groups():
    """Batches beyond 16384 query problems go out in slices of whole groups: with G = 3 a slice holds 16383."""
    desc = _descriptor(128, 128, 64, "bf16", batch=3 * 5500)
    for G, slices in ((1, 2), (3, 2), (8250, 2), (16500, None)):
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(KT.forward))
        if slices is None:
            with pytest.raises(mfa.MFAError):
                kernel.launchCount(_constants(desc, G))
        else:
            assert kernel.launchCount(_constants(desc, G)) == slices
    desc = _descriptor(128, 128, 64, "bf16", batch=2 * 16383)
    assert mfa.AttentionKernel(desc.kernelDescriptor(KT.forward)).launchCount(_constants(desc, 16383)) == 2
    assert mfa.AttentionKernel(desc.kernelDescriptor(KT.forward)).launchCount(_constants(desc, 2)) == 2


def test_group_is_not_part_of_the_kernel_or_its_cache_key():
    for mode in ("bf16", "fp32"):
        desc = _descriptor(512, 512, 128, mode, batch=8)
        for t in KT:
            first = mfa.AttentionKernel.cached(desc, t)
            size = mfa.AttentionKernel.cacheSize()
            names = set()
            for G in (0, 1, 2, 4, 8):
                _constants(desc, G)
                k = mfa.AttentionKernel.cached(desc, t)
                assert k._handle.value == first._handle.value
                names.add(k.sourceName())
            assert mfa.AttentionKernel.cacheSize() == size and names == {first.sourceName()}


def test_struct_layout_and_version():
    import ctypes
    assert ctypes.sizeof(mfa._CFunctionConstants) == 16 and mfa._CFunctionConstants.kv_group.offset == 12
    assert ctypes.sizeof(mfa._CDescriptor) == 24
    assert " 0.5 " in mfa.version() and "grouped K/V" in mfa.version()


def test_cpp_host_mirror_with_kv_group_compiles_and_links(tmp_path):
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  AttentionDescriptor d;
  d.lowPrecisionInputs = true;
  d.matrixDimensions = MatrixDimensions{2048, 1024, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  d.batchCount = 32;
  mfa_function_constants_t constants;
  constants.kv_group = 7;
  d.setFunctionConstants(constants);
  const unsigned reset = constants.kv_group;
  kvGroup(constants) = 16;
  AttentionKernel k(d.kernelDescriptor(AttentionKernelType::backwardKeyValue));
  std::printf("%u %u %u %zu\n", reset, constants.kv_group, k.gridSize(constants), sizeof(mfa_function_constants_t));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split()
    import ctypes
    assert out[:3] == ["0", "16", str(8 * 2)], out
    assert int(out[3]) == ctypes.sizeof(mfa._CFunctionConstants)


def test_grouped_head_partition():
    from mfa_b200.sharding import head_partition
    for total, G in ((64, 8), (32, 4), (24, 3), (8, 8), (12, 1)):
        for world in (1, 2, 3, 4, 8):
            owned = []
            for rank in range(world):
                start, count = head_partition(total, world, rank, kv_group=G)
                assert start % G == 0 and count % G == 0
                # the rank's K/V heads are the plain partition of the total / G K/V heads
                assert (start // G, count // G) == head_partition(total // G, world, rank)
                owned.extend(range(start, start + count))
            assert owned == list(range(total))
    assert head_partition(64, 8, 3) == head_partition(64, 8, 3, kv_group=1)
    with pytest.raises(ValueError):
        head_partition(10, 2, 0, kv_group=4)
    with pytest.raises(ValueError):
        head_partition(8, 2, 0, kv_group=0)


# ------------------------------------------------------------------------------------------------ GPU
def run(desc, G, inputs, types=tuple(KT), edit=None, raw=False):
    """Runs `types` with kvGroup = G on the current device: the harness's buffers (random out-of-bounds tails on the
    inputs, NaN-poisoned outputs whose tails must survive), with K, V, dK, dV sized batch / G.  `edit(kernel
    descriptor)` may change the split policy.  Returns {name: float32 array}: L / D in the oracle's units unless raw."""
    import torch
    from tests.attention_harness import _device_buffer
    R, C, D = desc.matrixDimensions
    B = desc.batchCount
    tQ, tK, tV, tO = desc.transposeState
    transposed = {Op.Q: tQ, Op.K: tK, Op.V: tV, Op.O: tO, Op.dO: tO, Op.dV: tV, Op.dK: tK, Op.dQ: tQ}
    prec = desc.memoryPrecisions
    rng = np.random.default_rng(12345)
    dev = {}
    for op, a in inputs.items():
        a = np.asarray(a, np.float32)
        if transposed[op]:
            a = np.ascontiguousarray(np.swapaxes(a, -1, -2))
        dev[op] = _device_buffer(oracle.encode(a, int(prec[op])), rng, int(prec[op]))
    kv = B // max(G, 1)   # K/V problems (G = 0: ungrouped)
    counts = {Op.O: B * R * D, Op.L: B * R, Op.D: B * R, Op.dQ: B * R * D, Op.dV: kv * C * D, Op.dK: kv * C * D}
    for op, n in counts.items():
        dev[op] = (torch.full((2 * n,), float("nan"), device="cuda") if prec[op] == P.FP32 else
                   torch.full((2 * n,), -1, dtype=torch.int16, device="cuda"))
    c = mfa.FunctionConstantValues()
    desc.setFunctionConstants(c)
    c.kvGroup = G
    ptrs = {op: t.data_ptr() for op, t in dev.items()}
    produced = {KT.forward: (Op.O, Op.L), KT.backwardQuery: (Op.D, Op.dQ), KT.backwardKeyValue: (Op.dV, Op.dK)}
    out = {}
    for t in KT:
        if t not in types:
            continue
        kd = desc.kernelDescriptor(t)
        if edit is not None:
            edit(kd)
        mfa.AttentionKernel(kd).encode(c, ptrs)
        for op in produced[t]:
            out[op] = None
    torch.cuda.synchronize()
    result = {}
    for op in out:
        n = counts[op]
        a = dev[op].cpu().numpy()
        vals, tail = a[:n], a[n:]
        if a.dtype == np.float32:
            assert np.isnan(tail).all(), f"a kernel wrote past the end of {op.name}"
        else:
            assert (tail == -1).all(), f"a kernel wrote past the end of {op.name}"
            vals = oracle.decode(vals.view(np.uint16), int(prec[op]))
        if op in (Op.L, Op.D):
            vals = vals.reshape(B, R)
        else:
            heads, seq = (B, R) if op in (Op.O, Op.dQ) else (kv, C)
            vals = (np.swapaxes(vals.reshape(heads, D, seq), -1, -2) if transposed[op] else vals.reshape(heads, seq, D))
        result[op.name] = np.ascontiguousarray(vals, np.float32)
    if not raw:
        if "L" in result:
            result["L"] = result["L"] / np.float32(LOG2E)
        if "D" in result:
            result["D"] = result["D"] * np.float32(np.sqrt(D))
    return result


def _check_reference(desc, G, out, ref, V, mode):
    """The backward suites' tolerances (tests/test_causal.py): check_O for O, 1e-3 / 2e-5 for L, 5e-2 and a relative RMS
    bound for the gradients; dK / dV sum G heads' terms, so their max-abs bound grows with sqrt(G)."""
    from tests.attention_harness import check
    from tests.test_tcgen05_backward import _rel_rms
    from tests.test_tcgen05_forward import check_O
    R, C, D = desc.matrixDimensions
    e = max(0, R - C) if desc.causal else 0
    assert np.isposinf(out["L"][:, :e]).all() and np.isfinite(out["L"][:, e:]).all()
    for name in ("O", "D", "dQ", "dK", "dV"):
        assert np.isfinite(out[name]).all(), name
    if mode == "fp32":
        check(ref["O"], out["O"], 2e-5, "O")
        check(ref["L"][:, e:], out["L"][:, e:], 2e-5, "L")
        for name in ("D", "dQ", "dK", "dV"):
            check(ref[name], out[name], 2e-5 * (np.sqrt(G) if name in ("dK", "dV") else 1), name)
        return
    check_O(ref["O"], out["O"], V, mode == "bf16")
    check(ref["L"][:, e:], out["L"][:, e:], 1e-3, "L")
    check(ref["D"], out["D"], 1e-1, "D")
    bound = 2.5e-3 if mode == "bf16" else 3e-4
    if min(R, C, D) < 16 or C < 32:
        bound *= 1.5
    for name in ("dQ", "dK", "dV"):
        check(ref[name], out[name], 5e-2 * (np.sqrt(G) if name in ("dK", "dV") else 1), name)
        rel = _rel_rms(out[name], ref[name])
        assert rel <= bound, f"{name}: relative RMS error {rel:.3e} > {bound}"


def _grouped_against_expanded(R, C, D, mode, B, G, causal=False, transpose=(False,) * 4, edit=None, seed=0):
    desc = _descriptor(R, C, D, mode, batch=B, causal=causal, transpose=transpose)
    inputs = _inputs(desc, G, seed)
    grouped = run(desc, G, inputs, edit=edit, raw=True)
    expanded = run(desc, 1, expand(inputs, G), edit=edit, raw=True)
    # forward and dQ: the same plan and arithmetic on the same values
    for name in ("O", "L", "D", "dQ"):
        assert grouped[name].tobytes() == expanded[name].tobytes(), f"{name} differs from the expanded K/V call"
    # dK / dV: the group sum, accumulated in one CTA, against the per-head results summed afterwards
    for name in ("dK", "dV"):
        summed = expanded[name].astype(np.float64).reshape(B // G, G, C, D).sum(axis=1)
        scale = max(float(np.abs(summed).max()), 1e-30)
        err = float(np.abs(grouped[name] - summed).max())
        assert err <= 2e-6 * G * scale, f"{name}: {err:.3e} from the sum of the expanded call's gradients"
    # deterministic: no atomics, every split partial written
    again = run(desc, G, inputs, edit=edit, raw=True)
    for name, a in grouped.items():
        assert again[name].tobytes() == a.tobytes(), name
    out = dict(grouped)
    out["L"] = out["L"] / np.float32(LOG2E)
    out["D"] = out["D"] * np.float32(np.sqrt(D))
    _check_reference(desc, G, out, reference(inputs, G, causal), inputs[Op.V], mode)
    return desc


CASES = [  # (R, C, D, mode, batch, G, causal, transpose)
    (200, 333, 64, "bf16", 4, 2, True, None),          # causal, R < C
    (130, 257, 128, "bf16", 6, 3, False, None),        # G not a power of two
    (128, 192, 64, "fp16", 16, 8, True, None),
    (96, 160, 128, "bf16", 5, 5, False, None),         # MQA: G = batch
    (300, 130, 64, "bf16", 4, 2, True, None),          # causal, R > C: rows that see no key
    (130, 200, 256, "bf16", 4, 2, True, None),         # D = 256 (split-D dK/dV)
    (256, 320, 256, "fp16", 6, 3, False, None),
    (100, 150, 40, "bf16", 4, 2, False, None),         # D % 8 != 0: staged
    (100, 150, 40, "reference", 6, 3, True, None),
    (136, 200, 128, "bf16", 6, 3, False, (True,) * 4),  # transposed operands: staged
    (136, 200, 64, "fp16", 4, 2, True, (False, True, True, False)),
    (64, 128, 64, "bf16", 3, 3, False, None),          # 1, 2, 3 query blocks per head: the ring crosses heads
    (128, 128, 128, "bf16", 3, 3, True, None),         # at both parities
    (192, 256, 64, "fp16", 2, 2, False, None),
    (256, 256, 64, "reference", 4, 2, False, None),    # FP16 + BF16 dO, converted on chip (small grid)
    (128, 1024, 64, "reference", 36, 2, True, None),   # ... converted in a pass of its own (> one wave of CTAs)
    (100, 77, 300, "fp32", 4, 2, True, None),          # SIMT FP32 family
    (64, 64, 32, "fp32", 6, 3, False, None),
    (130, 70, 160, "fp32", 3, 3, False, None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode,B,G,causal,transpose", CASES)
def test_grouped_matches_expanded_and_reference(R, C, D, mode, B, G, causal, transpose):
    desc = _grouped_against_expanded(R, C, D, mode, B, G, causal, transpose or (False,) * 4, seed=R + C + D + G)
    assert desc.kernelDescriptor(KT.forward).backend == (mfa.Backend.simtFP32 if mode == "fp32" else mfa.Backend.tcgen05)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_encode_rejects_invalid_groups(mode):
    desc = _descriptor(128, 128, 64, mode, batch=12)
    for t in KT:
        for G in (5, 16385):
            with pytest.raises(mfa.MFAError) as e:
                mfa.AttentionKernel(desc.kernelDescriptor(t)).encode(_constants(desc, G), {})
            assert e.value.status == -2 and "kv_group" in e.value.message


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode,causal", [(1024, 128, 128, "bf16", False), (1024, 128, 128, "bf16", True),
                                               (640, 64, 256, "fp16", True), (700, 100, 64, "reference", False)])
def test_split_dkdv_grid_over_one_kv_head(R, C, D, mode, causal):
    """One K/V head and few keys: a handful of dK/dV CTAs, so each head's query blocks are split into ranges (the same
    ranges for every head of the group) and summed by sum_splits; causal ranges can lie wholly before the tile."""
    G = 4
    desc = _descriptor(R, C, D, mode, batch=G, causal=causal)
    c = _constants(desc, G)
    assert mfa.AttentionKernel(desc.kernelDescriptor(KT.backwardKeyValue)).launchCount(c) == 2
    _grouped_against_expanded(R, C, D, mode, G, G, causal, seed=R + D)


@pytest.mark.gpu
@pytest.mark.parametrize("G", [8, 3])
def test_batches_beyond_one_launch_slice(G):
    """16 K/V heads past the first slice: the slices hold whole groups, their K/V offsets are h0 / G, and launchCount
    equals the kernels a torch.profiler trace of encode() records."""
    R, C, D = 16, 24, 64
    B = (16384 // G + 16) * G
    desc = _descriptor(R, C, D, "bf16", batch=B, causal=True)
    inputs = _inputs(desc, G, seed=G)
    out = run(desc, G, inputs)
    Q, K, V, dO = (inputs[op].astype(np.float64) for op in (Op.Q, Op.K, Op.V, Op.dO))
    Kq, Vq = np.repeat(K, G, axis=0), np.repeat(V, G, axis=0)
    S = np.einsum("brd,bcd->brc", Q, Kq) / np.sqrt(D)
    S = np.where(causal_mask(R, C)[None], S, -np.inf)
    Pm = np.exp(S - S.max(-1, keepdims=True))
    Pm /= Pm.sum(-1, keepdims=True)
    O = np.einsum("brc,bcd->brd", Pm, Vq)
    dS = Pm * (np.einsum("brd,bcd->brc", dO, Vq) - (dO * O).sum(-1)[..., None]) / np.sqrt(D)
    dK = np.einsum("brc,brd->bcd", dS, Q).reshape(B // G, G, C, D).sum(1)
    dV = np.einsum("brc,brd->bcd", Pm, dO).reshape(B // G, G, C, D).sum(1)
    assert np.abs(out["O"] - O).max() <= 2e-2
    assert np.abs(out["dK"] - dK).max() <= 5e-2 * np.sqrt(G) and np.abs(out["dV"] - dV).max() <= 5e-2 * np.sqrt(G)
    # launchCount against a torch.profiler trace, taken in a process of its own: the profiler's state is process-wide,
    # and the trace windows of other tests in this process must see exactly the history they see without this one
    code = f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests.test_kv_group import _trace_launches; " \
           f"print(json.dumps(_trace_launches({G})))"
    proc = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-4000:]
    for name, (launched, count) in json.loads(proc.stdout.strip().splitlines()[-1]).items():
        assert len(launched) == count >= 2, (name, launched, count)


def _trace_launches(G):
    """{kernel type: (names of the library's kernels a torch.profiler trace of one encode() records, launchCount)} for
    the sliced batch of test_batches_beyond_one_launch_slice."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    R, C, D = 16, 24, 64
    desc = _descriptor(R, C, D, "bf16", batch=(16384 // G + 16) * G, causal=True)
    c = _constants(desc, G)
    bufs = {op: torch.zeros(desc.operandElements(op) // (G if op in (Op.K, Op.V, Op.dK, Op.dV) else 1),
                            device="cuda", dtype=torch.float32 if desc.memoryPrecisions[op] == P.FP32 else torch.bfloat16)
            for op in (Op.Q, Op.K, Op.V, Op.O, Op.L, Op.D, Op.dO, Op.dV, Op.dK, Op.dQ)}
    ptrs = {op: b.data_ptr() for op, b in bufs.items()}
    out = {}
    for t in KT:
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(t))
        kernel.encode(c, ptrs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            # the trace can miss the first kernel of the window: a torch kernel goes first, and only the library's count
            bufs[Op.L].add_(0.0)
            torch.cuda.synchronize()
            kernel.encode(c, ptrs)
            torch.cuda.synchronize()
        launched = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                    and "mfa::" in e.name]
        out[t.name] = (launched, kernel.launchCount(c))
    return out


def _default_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(4))
def test_ungrouped_results_are_unchanged(case):
    """kvGroup 0 and 1 reproduce, bit for bit, what the library computed before grouped K/V existed: the SHA-256 of
    every output, recorded from that build on an H100 (grids chosen so that no plan depends on the SM count)."""
    import hashlib
    spec = _default_cases()[case]
    R, C, D = spec["R"], spec["C"], spec["D"]
    desc = _descriptor(R, C, D, spec["mode"], batch=spec["batch"], causal=spec["causal"])
    inputs = _inputs(desc, 1, spec["seed"])
    for G in (0, 1):
        out = run(desc, G, inputs, raw=True)
        for name, digest in spec["sha256"].items():
            assert hashlib.sha256(out[name].tobytes()).hexdigest() == digest, (G, name)
