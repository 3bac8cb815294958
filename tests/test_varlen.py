"""Packed variable-length sequences (AttentionKernel.encode(..., sequences=SequenceTable)): FlashAttention's cu_seqlens.

Sequence s owns query rows [qo[s], qo[s + 1]) and key rows [ko[s], ko[s + 1]) of every problem; Q, O, dO, dQ are
[H][row][D], L and D [H][row], K, V, dK, dV [H / G][column][D].  Within a sequence every output is attention on that
sequence alone (causal: bottom-right aligned per sequence), dK / dV summed over each K/V group.

The reference is tests/causal_oracle.attention_f64 per (sequence, head), pinned on the CPU against PyTorch's
scaled_dot_product_attention on the packed tokens with a block-diagonal mask.  On the GPU, every sequence's outputs must
equal bit for bit those of a separate call on that sequence alone (split off), a uniform table must equal the
fixed-length batched call, NaN in a neighbouring sequence must not change a sequence's outputs, rows past the table's
end keep their sentinels, and the results meet the backward suites' tolerances against the float64 reference."""
import ctypes

import numpy as np
import pytest

import mfa_b200 as mfa
import oracle
from tests.causal_oracle import attention_f64

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
LOG2E = 1.44269504089


def sequence_attention(Q, K, V, dO, causal):
    """attention_f64 of one (sequence, head), with the empty-sequence rules: Cs = 0 -> O = 0, L = +inf, D = dQ = 0."""
    R, D = Q.shape
    if K.shape[0] == 0:
        return {"O": np.zeros((R, D)), "L": np.full(R, np.inf), "D": np.zeros(R), "dQ": np.zeros((R, D)),
                "dK": np.zeros((0, D)), "dV": np.zeros((0, D))}
    return attention_f64(Q, K, V, dO, causal=causal)


def reference(inputs, G, qo, ko, causal):
    """float64 outputs in the packed layout: O, dQ [H][T][D], L, D [H][T], dK, dV [H / G][Tk][D] (rows past the
    table's end are zero)."""
    Q, K, V, dO = (np.asarray(inputs[op], np.float64) for op in (Op.Q, Op.K, Op.V, Op.dO))
    H, T, D = Q.shape
    out = {"O": np.zeros_like(Q), "dQ": np.zeros_like(Q), "L": np.zeros((H, T)), "D": np.zeros((H, T)),
           "dK": np.zeros_like(K), "dV": np.zeros_like(V)}
    for s in range(len(qo) - 1):
        q, k = slice(qo[s], qo[s + 1]), slice(ko[s], ko[s + 1])
        for h in range(H):
            r = sequence_attention(Q[h, q], K[h // G, k], V[h // G, k], dO[h, q], causal)
            for name in ("O", "dQ", "L", "D"):
                out[name][h, q] = r[name]
            out["dK"][h // G, k] += r["dK"]
            out["dV"][h // G, k] += r["dV"]
    return out


def _descriptor(R, C, D, mode, batch, causal, transpose=(False,) * 4, lowMid=False):
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


def _offsets(lengths):
    return [0] + list(np.cumsum(lengths).astype(int))


# ------------------------------------------------------------------------------------------------ CPU: the reference
@pytest.mark.parametrize("causal", [False, True])
def test_reference_matches_torch_sdpa_on_packed_tokens(causal):
    import torch
    rq, rk = [5, 0, 7, 3, 9], [6, 4, 0, 3, 5]   # an empty query sequence, an empty key sequence, Rs > Cs, Rs < Cs
    qo, ko = _offsets(rq), _offsets(rk)
    H, G, D = 4, 2, 8
    rng = np.random.default_rng(1)
    q, do = (rng.standard_normal((H, qo[-1], D)) for _ in range(2))
    k, v = (rng.standard_normal((H // G, ko[-1], D)) for _ in range(2))
    ref = reference({Op.Q: q, Op.K: k, Op.V: v, Op.dO: do}, G, qo, ko, causal)
    # block-diagonal mask over the packed tokens, bottom-right causal inside each block
    mask = np.zeros((qo[-1], ko[-1]), bool)
    for s in range(len(rq)):
        i, j = np.arange(rq[s])[:, None], np.arange(rk[s])[None, :]
        mask[qo[s]:qo[s + 1], ko[s]:ko[s + 1]] = (j <= i + rk[s] - rq[s]) if causal else True
    seen = mask.any(axis=1)   # rows that see no key are NaN in torch; the library's rule gives them O = 0
    tq, tk, tv = (torch.tensor(a, requires_grad=True) for a in (q, k, v))
    O = torch.nn.functional.scaled_dot_product_attention(tq, tk, tv, attn_mask=torch.tensor(mask), enable_gqa=True)
    O = torch.where(torch.tensor(seen)[None, :, None], O, torch.zeros_like(O))
    (O * torch.tensor(do)).sum().backward()
    for name, got in (("O", O.detach()), ("dQ", tq.grad), ("dK", tk.grad), ("dV", tv.grad)):
        assert np.abs(got.numpy() - ref[name]).max() <= 1e-10, name
    assert np.isposinf(ref["L"][:, ~seen]).all() and np.isfinite(ref["L"][:, seen]).all()
    assert (ref["dK"][:, ko[1]:ko[2]] == 0).all() or rq[1] != 0   # keys of the empty query sequence: zero gradient


# ------------------------------------------------------------------------------------------------ CPU: the API
def _constants(row, column, batch, G):
    c = mfa.FunctionConstantValues()
    c._c.row, c._c.column, c._c.batch_count, c._c.kv_group = row, column, batch, G
    return c


def test_sequence_table_layout():
    assert ctypes.sizeof(mfa.SequenceTable) == 32
    assert mfa.SequenceTable.row_offsets.offset == 16 and mfa.SequenceTable.column_offsets.offset == 24
    assert "packed sequences" in mfa.version() and " 0.5 " in mfa.version()


def test_grid_size_and_launch_count_of_packed_calls():
    """132 SMs without a device: grid (tiles of the longest sequence, heads, S); packed calls never split, and the dK/dV
    dO conversion runs as a pass of its own when the packed grid has more CTAs than SMs."""
    H, G = 8, 4
    for mode in ("bf16", "reference", "fp32"):
        desc = _descriptor(4096, 4096, 128, mode, H, False)
        kernels = {t: mfa.AttentionKernel(desc.kernelDescriptor(t)) for t in KT}
        par = {t: kernels[t].blockDimensions[0] for t in KT}
        c = _constants(4096, 3000, H, G)
        for S, max_row, max_column in ((1, 100, 100), (3, 1000, 700), (40, 4096, 3000)):
            table = mfa.SequenceTable(S, max_row, max_column, 16, 16)   # (not dereferenced on the host)
            assert kernels[KT.forward].gridSize(c, table) == -(-max_row // par[KT.forward]) * H * S
            assert kernels[KT.backwardQuery].gridSize(c, table) == -(-max_row // par[KT.backwardQuery]) * H * S
            kv_ctas = -(-max_column // par[KT.backwardKeyValue]) * (H // G) * S
            assert kernels[KT.backwardKeyValue].gridSize(c, table) == kv_ctas
            assert kernels[KT.forward].launchCount(c, table) == 1
            assert kernels[KT.backwardQuery].launchCount(c, table) == 1
            expected = 1 + (mode == "reference" and kv_ctas > 132)
            assert kernels[KT.backwardKeyValue].launchCount(c, table) == expected, (mode, S)


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_invalid_sequence_tables_are_rejected(mode):
    desc = _descriptor(256, 128, 64, mode, 4, False)
    c = _constants(256, 128, 4, 2)
    bad = [(None, "NULL sequence table"),
           (mfa.SequenceTable(2, 10, 10, 0, 16), "must not be NULL"),
           (mfa.SequenceTable(2, 10, 10, 16, 0), "must not be NULL"),
           (mfa.SequenceTable(0, 10, 10, 16, 16), "count 0"),
           (mfa.SequenceTable(65536, 10, 10, 16, 16), "count 65536"),
           (mfa.SequenceTable(2, 0, 10, 16, 16), "max_row 0"),
           (mfa.SequenceTable(2, 257, 10, 16, 16), "max_row 257"),
           (mfa.SequenceTable(2, 10, 0, 16, 16), "max_column 0"),
           (mfa.SequenceTable(2, 10, 129, 16, 16), "max_column 129")]
    for t in KT:
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(t))
        for table, message in bad:
            for call in (kernel.gridSize, kernel.launchCount):
                with pytest.raises(mfa.MFAError) as e:
                    if table is None:
                        out = ctypes.c_uint32()
                        fn = (mfa._lib.mfa_attention_kernel_grid_size_sequences if call == kernel.gridSize else
                              mfa._lib.mfa_attention_kernel_launch_count_sequences)
                        mfa._check(fn(kernel._handle, ctypes.byref(c._c), None, ctypes.byref(out)))
                    else:
                        call(c, table)
                assert e.value.status == -2 and message in e.value.message, (table, e.value.message)


def test_simt_family_rejects_transposed_packed_calls():
    desc = _descriptor(256, 128, 64, "fp32", 4, False, (False, True, False, False))
    c = _constants(256, 128, 4, 2)
    for t in KT:
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(t))
        assert kernel.gridSize(c) > 0   # fixed-length calls take transposed operands
        for call in (kernel.gridSize, kernel.launchCount):
            with pytest.raises(mfa.MFAError) as e:
                call(c, mfa.SequenceTable(2, 10, 10, 16, 16))
            assert e.value.status == -2 and "row-major" in e.value.message and "K is transposed" in e.value.message


def test_cpp_host_mirror_with_sequences(tmp_path):
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
  d.matrixDimensions = MatrixDimensions{4096, 4096, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  d.batchCount = 8;
  mfa_function_constants_t constants;
  d.setFunctionConstants(constants);
  kvGroup(constants) = 4;
  static int32_t fake[3];
  SequenceTable table{3, 1000, 700, fake, fake};
  AttentionKernel f(d.kernelDescriptor(AttentionKernelType::forward));
  AttentionKernel kv(d.kernelDescriptor(AttentionKernelType::backwardKeyValue));
  std::printf("%u %u %u %zu\n", f.gridSize(constants, table), kv.gridSize(constants, table), f.launchCount(constants, table),
              sizeof(mfa_sequence_table_t));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", root, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert out == [str(8 * 8 * 3), str(6 * 2 * 3), "1", str(ctypes.sizeof(mfa.SequenceTable))], out


# ------------------------------------------------------------------------------------------------ GPU
def _inputs(desc, G, T, Tk, seed):
    D = desc.matrixDimensions[2]
    H = desc.batchCount
    rng = np.random.default_rng(seed)
    x = {Op.Q: rng.standard_normal((H, T, D)), Op.K: rng.standard_normal((H // G, Tk, D)),
         Op.V: rng.standard_normal((H // G, Tk, D)), Op.dO: rng.standard_normal((H, T, D))}
    prec = desc.memoryPrecisions
    return {op: oracle.roundtrip(a.astype(np.float32), int(prec[op])) for op, a in x.items()}


def _transposed(desc):
    tQ, tK, tV, tO = desc.transposeState
    return {Op.Q: tQ, Op.K: tK, Op.V: tV, Op.O: tO, Op.dO: tO, Op.dV: tV, Op.dK: tK, Op.dQ: tQ}


def run_packed(desc, G, inputs, qo, ko, max_row=None, max_column=None, edit=None, graph_tables=None):
    """Packed encode of forward, dQ and dK/dV with row = T, column = Tk (the inputs' rows).  Inputs carry random tails
    past their buffers, outputs are NaN sentinels (also past the table's end, which must survive).  Transposed operands
    are stored [H][D][rows].  graph_tables = (qo, ko): the encodes are captured into a CUDA graph with the first table,
    and the graph is replayed after the device tables were overwritten with these.  Returns raw outputs {name: float32
    array} in the packed [H][rows][D] layout."""
    import torch
    from tests.attention_harness import _device_buffer
    H, T, D = inputs[Op.Q].shape
    Tk = inputs[Op.K].shape[1]
    prec = desc.memoryPrecisions
    transposed = _transposed(desc)
    rng = np.random.default_rng(12345)
    dev = {}
    for op, a in inputs.items():
        a = np.asarray(a, np.float32)
        if transposed[op]:
            a = np.ascontiguousarray(np.swapaxes(a, -1, -2))
        dev[op] = _device_buffer(oracle.encode(a, int(prec[op])), rng, int(prec[op]))
    counts = {Op.O: H * T * D, Op.L: H * T, Op.D: H * T, Op.dQ: H * T * D, Op.dV: H // G * Tk * D,
              Op.dK: H // G * Tk * D}
    for op, n in counts.items():
        dev[op] = (torch.full((2 * n,), float("nan"), device="cuda") if prec[op] == P.FP32 else
                   torch.full((2 * n,), -1, dtype=torch.int16, device="cuda"))
    tables = [torch.tensor(qo, dtype=torch.int32, device="cuda"), torch.tensor(ko, dtype=torch.int32, device="cuda")]
    rq, rk = np.diff(qo), np.diff(ko)
    table = mfa.SequenceTable(len(qo) - 1, max_row or max(1, int(rq.max())), max_column or max(1, int(rk.max())),
                              tables[0].data_ptr(), tables[1].data_ptr())
    c = _constants(T, Tk, H, G)
    ptrs = {op: t.data_ptr() for op, t in dev.items()}
    kernels = []
    for t in KT:
        kd = desc.kernelDescriptor(t)
        if edit is not None:
            edit(kd)
        kernels.append(mfa.AttentionKernel(kd))

    def encode_all(stream=0):
        for k in kernels:
            k.encode(c, ptrs, stream, sequences=table)

    encode_all()   # (outside any capture first: the library's workspaces grow on demand)
    torch.cuda.synchronize()
    if graph_tables is not None:
        stream = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            encode_all(stream.cuda_stream)
        for op in counts:
            dev[op].fill_(float("nan") if dev[op].dtype == torch.float32 else -1)
        for device_table, new in zip(tables, graph_tables):
            device_table.copy_(torch.tensor(new, dtype=torch.int32))
        g.replay()
        torch.cuda.synchronize()
    out = {}
    for op, n in counts.items():
        a = dev[op].cpu().numpy()
        vals, tail = a[:n], a[n:]
        if a.dtype == np.float32:
            assert np.isnan(tail).all(), f"a kernel wrote past the end of {op.name}"
        else:
            assert (tail == -1).all(), f"a kernel wrote past the end of {op.name}"
            vals = oracle.decode(vals.view(np.uint16), int(prec[op]))
        shape = {Op.L: (H, T), Op.D: (H, T), Op.O: (H, T, D), Op.dQ: (H, T, D)}.get(op, (H // G, Tk, D))
        if op not in (Op.L, Op.D) and transposed[op]:
            vals = np.swapaxes(vals.reshape(shape[0], D, shape[1]), -1, -2)
        out[op.name] = np.ascontiguousarray(vals.reshape(shape), np.float32)
    return out


def _check_against_reference(out, ref, qo, ko, mode, G, D):
    from tests.test_tcgen05_backward import _rel_rms
    T, Tk = qo[-1], ko[-1]
    got = {n: out[n][:, :T] if n in ("O", "dQ", "L", "D") else out[n][:, :Tk] for n in out}
    got["L"] = got["L"] / np.float32(LOG2E)
    got["D"] = got["D"] * np.float32(np.sqrt(D))
    ref = {n: ref[n][:, :T] if n in ("O", "dQ", "L", "D") else ref[n][:, :Tk] for n in ref}
    inf = np.isposinf(ref["L"])
    assert (np.isposinf(got["L"]) == inf).all(), "rows that see no key get L = +inf"
    got["L"][inf] = 0.0
    ref["L"][inf] = 0.0
    for name in got:
        assert np.isfinite(got[name]).all(), name
    fp32 = mode == "fp32"
    bars = {"O": 2e-5 if fp32 else (2e-2 if mode == "bf16" else 5e-3), "L": 2e-5 if fp32 else 1e-3,
            "D": 2e-5 if fp32 else 1e-1}
    for name, bar in bars.items():
        err = float(np.abs(got[name] - ref[name]).max())
        assert err <= bar, f"{name}: {err:.3e} > {bar}"
    for name in ("dQ", "dK", "dV"):
        bar = (2e-5 if fp32 else 5e-2) * (np.sqrt(G) if name != "dQ" else 1)
        err = float(np.abs(got[name] - ref[name]).max())
        assert err <= bar, f"{name}: {err:.3e} > {bar}"
        if not fp32 and np.abs(ref[name]).max() > 0:
            rel = _rel_rms(got[name], ref[name])
            assert rel <= (2.5e-3 if mode == "bf16" else 3e-4) * 1.5, f"{name}: relative RMS {rel:.3e}"


def _check_sentinels(out, qo, ko):
    """Rows past the table's end keep their sentinels (0xFFFF in 16-bit outputs, which decodes to NaN)."""
    for name in ("O", "dQ", "L", "D"):
        assert np.isnan(out[name][:, qo[-1]:]).all(), name
    for name in ("dK", "dV"):
        assert np.isnan(out[name][:, ko[-1]:]).all(), name


def _split_off(kd):
    kd.splitPolicy = (0, 1)


def _per_sequence_bitwise(desc, G, inputs, out, qo, ko):
    """Every sequence with Rs, Cs >= 1 against a separate fixed-length call on that sequence alone, split off."""
    H, _, D = inputs[Op.Q].shape
    from tests.test_kv_group import run
    for s in range(len(qo) - 1):
        Rs, Cs = qo[s + 1] - qo[s], ko[s + 1] - ko[s]
        if Rs == 0 or Cs == 0:
            continue
        single = _descriptor(Rs, Cs, D, _mode_of(desc), H, desc.causal, desc.transposeState)
        part = {op: a[:, qo[s]:qo[s + 1]] if op in (Op.Q, Op.dO) else a[:, ko[s]:ko[s + 1]] for op, a in inputs.items()}
        alone = run(single, G, part, edit=_split_off, raw=True)
        for name in ("O", "L", "D", "dQ"):
            assert alone[name].tobytes() == np.ascontiguousarray(out[name][:, qo[s]:qo[s + 1]]).tobytes(), (s, name)
        for name in ("dK", "dV"):
            assert alone[name].tobytes() == np.ascontiguousarray(out[name][:, ko[s]:ko[s + 1]]).tobytes(), (s, name)


def _mode_of(desc):
    prec = desc.memoryPrecisions
    if prec[Op.Q] == P.FP32:
        return "fp32"
    if prec[Op.dO] != prec[Op.Q]:
        return "reference"
    return "bf16" if prec[Op.Q] == P.BF16 else "fp16"


LENGTHS = {  # (query lengths, key lengths)
    "edges": ([1, 63, 64, 65, 127, 129, 1000], [1, 63, 64, 65, 127, 129, 1000]),
    "empty": ([70, 0, 130, 40], [90, 50, 0, 40]),             # a 0-length query sequence, a 0-length key sequence
    "taller": ([200, 65, 129], [100, 64, 7]),                 # Rs > Cs (causal: rows that see no key)
    "long_among_short": ([3, 5, 900, 2, 7, 1, 4], [3, 5, 900, 2, 7, 1, 4]),
}
CASES = [  # (mode, D, causal, G, lengths)
    ("bf16", 128, True, 4, "edges"), ("bf16", 128, False, 1, "empty"), ("bf16", 64, True, 1, "taller"),
    ("fp16", 64, False, 4, "edges"), ("fp16", 256, True, 4, "empty"), ("bf16", 256, False, 1, "long_among_short"),
    ("reference", 128, True, 4, "taller"), ("reference", 64, False, 1, "long_among_short"),
    ("bf16", 72, True, 4, "empty"), ("fp32", 64, True, 4, "taller"), ("fp32", 72, False, 1, "empty"),
    ("fp32", 128, True, 1, "long_among_short"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,G,lengths", CASES)
def test_packed_matches_reference_and_separate_calls(mode, D, causal, G, lengths):
    rq, rk = LENGTHS[lengths]
    qo, ko = _offsets(rq), _offsets(rk)
    H = 4
    T, Tk = qo[-1] + 9, ko[-1] + 5   # rows past the table's end: never read, never written
    desc = _descriptor(T, Tk, D, mode, H, causal)
    inputs = _inputs(desc, G, T, Tk, seed=D + G + len(rq))
    out = run_packed(desc, G, inputs, qo, ko)
    _check_sentinels(out, qo, ko)
    _check_against_reference(out, reference(inputs, G, qo, ko, causal), qo, ko, mode, G, D)
    _per_sequence_bitwise(desc, G, inputs, out, qo, ko)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,causal", [("bf16", False), ("bf16", True), ("reference", True), ("fp32", False)])
def test_uniform_table_equals_the_batched_call(mode, causal):
    """G = 1, S sequences of L rows over H heads are the fixed-length call with batch H * S: the same memory."""
    from tests.test_kv_group import run
    H, S, L, D = 3, 4, 192, 128
    desc = _descriptor(S * L, S * L, D, mode, H, causal)
    inputs = _inputs(desc, 1, S * L, S * L, seed=5)
    qo = [s * L for s in range(S + 1)]
    out = run_packed(desc, 1, inputs, qo, qo)
    batched = _descriptor(L, L, D, mode, H * S, causal)
    fixed = run(batched, 1, {op: a.reshape(H * S, L, D) for op, a in inputs.items()}, edit=_split_off, raw=True)
    for name, a in fixed.items():
        assert a.tobytes() == out[name].reshape(a.shape).tobytes(), name


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "reference", "fp32"])
def test_nan_in_a_neighbouring_sequence_does_not_leak(mode):
    rq = rk = [100, 65, 130]
    qo, ko = _offsets(rq), _offsets(rk)
    G, H, D = 2, 4, 128
    desc = _descriptor(qo[-1], ko[-1], D, mode, H, True)
    inputs = _inputs(desc, G, qo[-1], ko[-1], seed=3)
    clean = run_packed(desc, G, inputs, qo, ko)
    poisoned = {op: a.copy() for op, a in inputs.items()}
    for op in (Op.Q, Op.dO):
        poisoned[op][:, qo[1]:qo[2]] = np.nan
    for op in (Op.K, Op.V):
        poisoned[op][:, ko[1]:ko[2]] = np.inf
    dirty = run_packed(desc, G, poisoned, qo, ko)
    for s in (0, 2):
        for name in ("O", "L", "D", "dQ"):
            assert clean[name][:, qo[s]:qo[s + 1]].tobytes() == dirty[name][:, qo[s]:qo[s + 1]].tobytes(), (s, name)
        for name in ("dK", "dV"):
            assert clean[name][:, ko[s]:ko[s + 1]].tobytes() == dirty[name][:, ko[s]:ko[s + 1]].tobytes(), (s, name)


@pytest.mark.gpu
def test_packed_encode_replays_in_a_cuda_graph_with_new_table_contents():
    """A graph captured with one table replays with whatever the device tables hold: the same count and maxima, new
    lengths, and the same results as an eager call on the new table."""
    first, second = ([130, 7, 300], [64, 200, 300]), ([300, 100, 37], [120, 300, 144])
    T, Tk = 450, 600
    desc = _descriptor(T, Tk, 128, "bf16", 8, True)
    inputs = _inputs(desc, 4, T, Tk, seed=9)
    tables = [(_offsets(rq), _offsets(rk)) for rq, rk in (first, second)]
    eager = run_packed(desc, 4, inputs, *tables[1], max_row=300, max_column=300)
    graphed = run_packed(desc, 4, inputs, *tables[0], max_row=300, max_column=300, graph_tables=tables[1])
    for name, a in eager.items():
        assert a.tobytes() == graphed[name].tobytes(), name


STAGED = [  # (mode, D, causal, G, transpose): operands staged row-major with pad8(D) columns and copied back
    ("bf16", 60, True, 2, (False,) * 4), ("reference", 60, False, 1, (False,) * 4),
    ("bf16", 128, True, 2, (True,) * 4), ("fp16", 64, False, 1, (False, True, True, False)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,D,causal,G,transpose", STAGED)
def test_staged_operands_keep_rows_outside_the_sequences(mode, D, causal, G, transpose):
    """Head dimensions that are not multiples of 8 and transposed operands go through the staging copies; the copy-back
    writes only the sequences' rows, so sentinel rows past the table's end survive, also with max_row / max_column
    below the buffers' rows."""
    # (transposed operands run on the tensor cores when their rows are a multiple of 8, here and in the separate calls)
    rq, rk = [72, 0, 128, 40], [88, 48, 0, 40]
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 72, ko[-1] + 72   # more rows past the table's end than any tile covers
    desc = _descriptor(T, Tk, D, mode, 4, causal, transpose)
    inputs = _inputs(desc, G, T, Tk, seed=D + G)
    assert desc.kernelDescriptor(KT.forward).backend == mfa.Backend.tcgen05
    out = run_packed(desc, G, inputs, qo, ko)
    _check_sentinels(out, qo, ko)
    _check_against_reference(out, reference(inputs, G, qo, ko, causal), qo, ko, mode, G, D)
    _per_sequence_bitwise(desc, G, inputs, out, qo, ko)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_encode_rejects_invalid_sequence_tables(mode):
    import torch
    desc = _descriptor(256, 128, 64, mode, 4, False)
    offsets = torch.zeros(3, dtype=torch.int32, device="cuda")
    p = offsets.data_ptr()
    for t in KT:
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(t))
        for c, table, message in ((_constants(256, 128, 4, 2), mfa.SequenceTable(0, 10, 10, p, p), "count 0"),
                                  (_constants(256, 128, 4, 2), mfa.SequenceTable(2, 10, 129, p, p), "max_column 129"),
                                  (_constants(256, 128, 4, 2), mfa.SequenceTable(2, 10, 10, 0, p), "must not be NULL"),
                                  (_constants(0, 128, 4, 2), mfa.SequenceTable(2, 10, 10, p, p), "at least 1")):
            with pytest.raises(mfa.MFAError) as e:
                kernel.encode(c, {}, sequences=table)
            assert e.value.status == -2 and message in e.value.message, e.value.message


@pytest.mark.gpu
def test_launch_count_matches_a_profiler_trace():
    """launchCount(sequences=) against the kernels a torch.profiler trace of one packed encode records: unstaged and
    staged operands, and the reference policy's BF16 dO converted on chip (small grid) or in a pass of its own."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = f"import json, sys; sys.path.insert(0, {root!r}); from tests.test_varlen import _trace_launches; " \
           f"print(json.dumps(_trace_launches()))"
    proc = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-4000:]
    results = json.loads(proc.stdout.strip().splitlines()[-1])
    for name, (launched, count) in results.items():
        assert len(launched) == count, (name, launched, count, results)
    assert results["reference D=64 S=40 backwardKeyValue"][1] == 2    # > 132 CTAs: the conversion pass
    assert results["reference D=64 S=2 backwardKeyValue"][1] == 1     # converted on chip
    assert results["bf16 D=60 S=2 forward"][1] == 1 + 4               # Q, K, V staged, O copied back


def _trace_launches():
    """{case: (names of the library's kernels a torch.profiler trace of one packed encode records, launchCount)}, run
    in a process of its own (the profiler's state is process-wide)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for mode, D, S in (("reference", 64, 40), ("reference", 64, 2), ("bf16", 60, 2), ("bf16", 128, 3)):
        lengths = [130 + 3 * s for s in range(S)]   # S = 40: 2 dK/dV tiles x 4 K/V heads x 40 > 132 CTAs
        qo = _offsets(lengths)
        T, H, G = qo[-1], 8, 2
        desc = _descriptor(T, T, D, mode, H, True)
        inputs = _inputs(desc, G, T, T, seed=S)
        prec = desc.memoryPrecisions
        bufs = {}
        for op in (Op.Q, Op.K, Op.V, Op.O, Op.L, Op.D, Op.dO, Op.dV, Op.dK, Op.dQ):
            heads = H // G if op in (Op.K, Op.V, Op.dK, Op.dV) else H
            n = heads * T * (1 if op in (Op.L, Op.D) else D)
            dtype = torch.float32 if prec[op] == P.FP32 else (torch.bfloat16 if prec[op] == P.BF16 else torch.float16)
            bufs[op] = torch.zeros(n, device="cuda", dtype=dtype)
        for op in (Op.Q, Op.K, Op.V, Op.dO):
            bufs[op].copy_(torch.tensor(inputs[op].reshape(-1)))
        ptrs = {op: b.data_ptr() for op, b in bufs.items()}
        table_d = torch.tensor(qo, dtype=torch.int32, device="cuda")
        table = mfa.SequenceTable(S, max(lengths), max(lengths), table_d.data_ptr(), table_d.data_ptr())
        c = _constants(T, T, H, G)
        for t in KT:
            kernel = mfa.AttentionKernel(desc.kernelDescriptor(t))
            kernel.encode(c, ptrs, sequences=table)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                # the trace can miss the first kernel of the window: a torch kernel goes first, and only the library's count
                bufs[Op.L].add_(0.0)
                torch.cuda.synchronize()
                kernel.encode(c, ptrs, sequences=table)
                torch.cuda.synchronize()
            launched = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                        and "mfa::" in e.name]
            out[f"{mode} D={D} S={S} {t.name}"] = (launched, kernel.launchCount(c, table))
    return out
