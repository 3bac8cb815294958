"""Causal attention (AttentionDescriptor.causal): the bottom-right aligned mask on the wgmma and SIMT kernels, forward,
dQ and dK/dV, against the causal reference of tests/causal_oracle.py.

With delta = C - R, query row i sees key j iff j <= i + delta.  Rows with no visible key (R > C, i < R - C) have
O = 0, L = +inf, D = 0, dQ = 0 exactly and add nothing to dK / dV.  Tolerances are the non-causal suites': check_O and
the L bounds of test_tcgen05_forward.py, the gradient bounds of test_tcgen05_backward.py, 2e-5 for the FP32 family."""
import os
import subprocess

import numpy as np
import pytest

import mfa_b200 as mfa
from tests.causal_oracle import Network, attention_f64, causal_mask

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _descriptor(R, C, D, mode="bf16", lowMid=False, batch=1, transpose=(False,) * 4, causal=True):
    """mode: "bf16" / "fp16" (all operands of that type), "reference" (FP16 Q/K/V, BF16 dO) or "fp32" (SIMT family)."""
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


def _network(desc, seed, causal=True):
    R, C, D = desc.matrixDimensions
    net = Network(R, C, D, seed=seed, threads=8, causal=causal)
    prec = desc.memoryPrecisions
    if prec[Op.Q] != P.FP32:
        net.round_inputs(int(prec[Op.Q]), int(prec[Op.dO]))
    return net


def _empty_rows(R, C):
    return max(0, R - C)


# ------------------------------------------------------------------------------------------------ CPU: the reference
def _row_by_row(net):
    """The causal problem as R unmasked ones: row i against its i + delta + 1 visible keys, on the C oracle."""
    import oracle
    R, C, D = net._dims()
    delta = C - R
    out = {"O": np.zeros((R, D)), "L": np.full(R, np.inf), "D": np.zeros(R), "dQ": np.zeros((R, D)),
           "dK": np.zeros((C, D)), "dV": np.zeros((C, D))}
    for i in range(R):
        k = i + delta + 1
        if k <= 0:
            continue
        row = oracle.Network(1, k, D)
        row.Q, row.dO = net.Q[i:i + 1].copy(), net.dO[i:i + 1].copy()
        row.K, row.V = net.K[:k].copy(), net.V[:k].copy()
        O, L = row.inferenceAttention(with_L=True)
        out["O"][i], out["L"][i], out["D"][i] = O[0], L[0], row.createDTerms()[0]
        out["dQ"][i] = row.derivativeQ()[0]
        out["dK"][:k] += row.derivativeK()
        out["dV"][:k] += row.derivativeV()
    return out


CPU_SHAPES = [(33, 33, 3), (64, 64, 40), (20, 45, 40), (17, 90, 64), (50, 18, 64), (40, 7, 3), (70, 70, 64)]


@pytest.mark.parametrize("R,C,D", CPU_SHAPES)
def test_causal_reference_matches_the_c_oracle_row_by_row(R, C, D):
    net = Network(R, C, D, seed=R + C + D, causal=True)
    ref = _row_by_row(net)
    got = attention_f64(net.Q, net.K, net.V, net.dO, causal=True)
    for name in ("O", "L", "D", "dQ", "dK", "dV"):
        e, a = ref[name], got[name]
        finite = np.isfinite(e)
        assert (np.isposinf(e) == np.isposinf(a)).all(), name
        scale = max(float(np.abs(e[finite]).max()), 1e-30)
        assert np.abs(e[finite] - a[finite]).max() <= 1e-5 * scale, name
    # the float32 interface the GPU tests use
    O, L = net.inferenceAttention(with_L=True)
    assert np.allclose(O, got["O"], atol=1e-6) and np.array_equal(np.isposinf(L), np.isposinf(got["L"]))
    assert np.allclose(net.derivativeK(), got["dK"], atol=1e-5 * np.abs(got["dK"]).max())
    e = _empty_rows(R, C)
    assert np.isposinf(L[:e]).all() and np.isfinite(L[e:]).all()
    assert (O[:e] == 0).all()
    assert (net.derivativeQ()[:e] == 0).all() and (net.createDTerms()[:e] == 0).all()


def test_unmasked_reference_is_the_c_oracle():
    """Without the mask the formulation is oracle_np's, and Network(causal=False) is the C oracle itself."""
    import oracle
    net = Network(45, 30, 24, seed=3)
    ref = {"O": net.inferenceAttention(), "dQ": net.derivativeQ(), "dK": net.derivativeK(), "dV": net.derivativeV()}
    got = attention_f64(net.Q, net.K, net.V, net.dO)
    for name, e in ref.items():
        assert np.abs(e - got[name]).max() <= 1e-5 * np.abs(e).max(), name
    plain = oracle.Network(45, 30, 24, seed=3)
    assert np.array_equal(plain.inferenceAttention(), ref["O"])


@pytest.mark.parametrize("R,C,D", [(48, 48, 16), (20, 61, 32), (61, 20, 8)])
def test_causal_reference_matches_torch_sdpa_with_an_explicit_mask(R, C, D):
    import torch
    net = Network(R, C, D, seed=7 * R + C, causal=True)
    got = attention_f64(net.Q, net.K, net.V, net.dO, causal=True)
    e = _empty_rows(R, C)
    q, k, v = (torch.tensor(np.asarray(x, np.float64), requires_grad=True) for x in (net.Q, net.K, net.V))
    mask = torch.tensor(causal_mask(R, C))
    O = torch.nn.functional.scaled_dot_product_attention(q[e:], k, v, attn_mask=mask[e:])
    (O * torch.tensor(np.asarray(net.dO[e:], np.float64))).sum().backward()
    assert np.abs(O.detach().numpy() - got["O"][e:]).max() <= 1e-10
    assert np.abs(q.grad.numpy()[e:] - got["dQ"][e:]).max() <= 1e-10
    assert np.abs(k.grad.numpy() - got["dK"]).max() <= 1e-10
    assert np.abs(v.grad.numpy() - got["dV"]).max() <= 1e-10
    if R == C:
        O2 = torch.nn.functional.scaled_dot_product_attention(q.detach(), k.detach(), v.detach(), is_causal=True)
        assert np.abs(O2.numpy() - got["O"]).max() <= 1e-10


def test_causal_gradients_match_finite_differences_of_the_masked_loss():
    R, C, D = 24, 37, 16
    net = Network(R, C, D, seed=5, causal=True)
    Q, K, V, dO = (np.asarray(x, np.float64) for x in (net.Q, net.K, net.V, net.dO))
    grads = attention_f64(Q, K, V, dO, causal=True)

    def loss(q, k, v):
        return float((dO * attention_f64(q, k, v, causal=True)["O"]).sum())

    h = 1e-6
    rng = np.random.default_rng(0)
    for name, grad in (("Q", "dQ"), ("K", "dK"), ("V", "dV")):
        for _ in range(6):
            x = {"Q": Q, "K": K, "V": V}
            i, d = int(rng.integers(x[name].shape[0])), int(rng.integers(D))
            plus, minus = ({n: a.copy() for n, a in x.items()} for _ in range(2))
            plus[name][i, d] += h
            minus[name][i, d] -= h
            fd = (loss(plus["Q"], plus["K"], plus["V"]) - loss(minus["Q"], minus["K"], minus["V"])) / (2 * h)
            assert abs(fd - grads[grad][i, d]) <= 1e-6 + 1e-5 * abs(fd), (name, i, d, fd, grads[grad][i, d])
    # the last key is visible to the last row only, and still gets a gradient
    assert np.abs(grads["dK"][C - 1]).max() > 0


# ------------------------------------------------------------------------------------------------ CPU: the API
def test_causal_defaults_off_and_reaches_every_kernel_descriptor():
    d = _descriptor(256, 256, 64, causal=False)
    assert mfa.AttentionDescriptor().causal is False
    for t in KT:
        assert d.kernelDescriptor(t).causal is False
    for mode in ("bf16", "fp32"):
        d = _descriptor(256, 300, 64, mode=mode)
        for t in KT:
            kd = d.kernelDescriptor(t)
            assert kd.causal is True
            kd.causal = False
            assert kd.causal is False


def test_unknown_causal_mode_is_rejected():
    d = _descriptor(128, 128, 64)
    d.causal = 2
    with pytest.raises(mfa.MFAError) as e:
        d.kernelDescriptor(KT.forward)
    assert e.value.status == -2
    kd = _descriptor(128, 128, 64).kernelDescriptor(KT.forward)
    kd.causal = 2
    with pytest.raises(mfa.MFAError) as e:
        mfa.AttentionKernel(kd)
    assert e.value.status == -2


def test_kernel_cache_keeps_causal_and_unmasked_kernels_apart():
    for mode in ("bf16", "fp32"):
        for t in KT:
            masked = mfa.AttentionKernel.cached(_descriptor(512, 512, 128, mode=mode, causal=True), t)
            plain = mfa.AttentionKernel.cached(_descriptor(512, 512, 128, mode=mode, causal=False), t)
            again = mfa.AttentionKernel.cached(_descriptor(512, 512, 128, mode=mode, causal=True), t)
            assert masked._handle.value != plain._handle.value and masked._handle.value == again._handle.value
            assert masked.sourceName() == plain.sourceName() + "_causal"
            assert not plain.sourceName().endswith("_causal")


def test_version_and_struct_layout():
    assert " 0.5 " in mfa.version()
    import ctypes
    # the request descriptor keeps its size (the field replaces a reserved byte)
    assert ctypes.sizeof(mfa._CDescriptor) == 24 and mfa._CDescriptor.causal.offset == 19


def test_cpp_host_mirror_with_causal_compiles_and_links(tmp_path):
    src = tmp_path / "host.cpp"
    src.write_text(r'''
#include <cstdio>
#include "metal-flash-attention_b200/host/FlashAttention.hpp"
using namespace FlashAttention;
int main() {
  AttentionDescriptor d;
  d.lowPrecisionInputs = true;
  d.matrixDimensions = MatrixDimensions{1024, 4096, 128};
  d.transposeState = TransposeState{false, false, false, false};
  d.inputPrecisionOverride = GEMMOperandPrecision::BF16;
  d.causal = true;
  AttentionKernelDescriptor kd = d.kernelDescriptor(AttentionKernelType::backwardKeyValue);
  AttentionKernel k(kd);
  AttentionKernel cached(d, AttentionKernelType::forward);
  kd.causal() = 0;
  AttentionKernel plain(kd);
  std::printf("%d %s %s %s %zu %zu\n", d.c().causal, k.sourceName().c_str(), cached.sourceName().c_str(),
              plain.sourceName().c_str(), sizeof(mfa_attention_descriptor_t), sizeof(mfa_attention_kernel_descriptor_t));
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(mfa.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lmfa_b200",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True).split()
    import ctypes
    assert out[:4] == ["1", "attention_backward_key_value_tcgen05<D=128>_causal", "attention_forward_tcgen05<D=128>_causal",
                       "attention_backward_key_value_tcgen05<D=128>"], out
    assert int(out[4]) == ctypes.sizeof(mfa._CDescriptor) and int(out[5]) == ctypes.sizeof(mfa._CKernelDescriptor)


# ------------------------------------------------------------------------------------------------ GPU
def _check_forward(desc, net, out, bf16, L_tol):
    from tests.attention_harness import check
    from tests.test_tcgen05_forward import check_O
    R, C, D = desc.matrixDimensions
    O, L = net.inferenceAttention(with_L=True)
    e = _empty_rows(R, C)
    assert np.isposinf(out["L"][..., :e]).all(), "rows with no visible key: L = +inf"
    assert (out["O"][..., :e, :] == 0).all(), "rows with no visible key: O = 0"
    assert np.isfinite(out["O"]).all() and np.isfinite(out["L"][..., e:]).all()
    if bf16 is None:
        check(O, out["O"], 2e-5, "O")
    else:
        check_O(O, out["O"], net.V, bf16)
    check(L, out["L"], L_tol, "L")


def _forward(R, C, D, mode, seed, lowMid=False, transpose=(False,) * 4):
    from tests.attention_harness import run_attention
    desc = _descriptor(R, C, D, mode, lowMid=lowMid, transpose=transpose)
    assert desc.kernelDescriptor(KT.forward).backend == (mfa.Backend.simtFP32 if mode == "fp32" else mfa.Backend.tcgen05)
    net = _network(desc, seed)
    out = run_attention(desc, net, types=[KT.forward])
    _check_forward(desc, net, out, None if mode == "fp32" else mode == "bf16",
                   2e-5 if mode == "fp32" else (7e-3 if lowMid else 1e-3))
    return out


def _backward(R, C, D, mode, seed, lowMid=False, transpose=(False,) * 4):
    from tests.attention_harness import run_attention, oracle_outputs, check
    from tests.test_tcgen05_backward import _rel_rms
    desc = _descriptor(R, C, D, mode, lowMid=lowMid, transpose=transpose)
    net = _network(desc, seed)
    out = run_attention(desc, net)
    ref = oracle_outputs(net)
    e = _empty_rows(R, C)
    for name in ("O", "D", "dQ", "dK", "dV"):
        assert np.isfinite(out[name]).all(), name
    assert np.isposinf(out["L"][:e]).all() and np.isfinite(out["L"][e:]).all()
    assert (out["D"][:e] == 0).all() and (out["dQ"][:e] == 0).all(), "rows with no visible key: D = 0, dQ = 0"
    if mode == "fp32":
        for name in ("O", "L", "D", "dV", "dK", "dQ"):
            check(ref[name], out[name], 2e-5, name)
        return out, ref
    # D of a row that sees a handful of keys carries P's 16-bit rounding undiluted (O is a mean of a few V rows): those
    # rows are held to the reference's bar (RectangularAttentionTest.swift:459-464), the others to the tighter one
    few = np.clip(np.arange(R) + (C - R) + 1, 0, C) < 16
    check(ref["D"][~few], out["D"][~few], 1e-1 if lowMid else 2e-2, "D")
    check(ref["D"][few], out["D"][few], 1e-1, "D (rows with < 16 visible keys)")
    bound = 2.5e-3 if mode == "bf16" else 3e-4
    if min(R, C, D) < 16 or C < 32:
        bound *= 1.5   # few terms per output element; under the mask key j (R >= C) gets only C - j of them
    if lowMid and mode != "bf16":
        bound = 2.5e-3
    for name in ("dV", "dK", "dQ"):
        check(ref[name], out[name], 5e-2, name)
        rel = _rel_rms(out[name], ref[name])
        assert rel <= bound, f"{name}: relative RMS error {rel:.3e} > {bound}"
    return out, ref


FORWARD_SHAPES = [
    (256, 256, 128), (128, 128, 64), (512, 384, 128), (256, 640, 64),   # aligned
    (200, 333, 128), (77, 129, 64), (1, 1, 8), (300, 17, 80), (129, 257, 72), (40, 500, 16),  # ragged edges
    (1024, 1024, 128), (640, 1280, 96),
    (256, 256, 256), (200, 333, 192), (384, 512, 136), (130, 70, 256), (1024, 1024, 256),   # 128 < D <= 256 kernel
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp16"])
@pytest.mark.parametrize("R,C,D", FORWARD_SHAPES)
def test_causal_forward_matches_the_causal_oracle(R, C, D, mode):
    _forward(R, C, D, mode, seed=R * 7 + C * 3 + D)


@pytest.mark.gpu
def test_causal_forward_fp16_L_storage():
    _forward(256, 256, 128, "bf16", seed=5, lowMid=True)
    _forward(300, 200, 64, "fp16", seed=6, lowMid=True)   # +inf L of the empty rows survives FP16 storage


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,bf16", [
    (4096, 4096, 128, True), (256, 2048, 64, False), (300, 2000, 128, True), (512, 1536, 96, True),
    (1, 4096, 128, False), (2048, 2048, 64, True), (129, 1024, 64, False), (64, 3000, 128, False),
    (256, 4096, 8, True), (100, 2560, 120, True), (384, 1024, 32, False), (640, 2048, 64, True)])
def test_causal_split_kv(R, C, D, bf16):
    """The split policy and launch count do not change with the mask; split ranges wholly past the diagonal of a tile
    leave L = -inf partials that the merge weighs 0."""
    desc = _descriptor(R, C, D, "bf16" if bf16 else "fp16")
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    assert mfa.AttentionKernel(desc.kernelDescriptor(KT.forward)).launchCount(constants) == 2
    _forward(R, C, D, "bf16" if bf16 else "fp16", seed=R + C + D)


@pytest.mark.gpu
def test_causal_split_kv_with_empty_rows():
    """R > C on a split grid: whole split ranges and whole rows see no key (L = +inf after the merge)."""
    import torch
    desc = _descriptor(384, 256, 64, "bf16")
    kd = desc.kernelDescriptor(KT.forward)
    kd.splitPolicy = (1, 4)      # edited: 3 query tiles x 4 key ranges of one block
    net = _network(desc, seed=17)
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    kernel = mfa.AttentionKernel(kd)
    assert kernel.launchCount(constants) == 2
    q, k, v = (torch.from_numpy(np.asarray(x, np.float32)).to(torch.bfloat16).cuda() for x in (net.Q, net.K, net.V))
    O = torch.full((384, 64), float("nan"), device="cuda")
    L = torch.full((384,), float("nan"), device="cuda")
    kernel.encode(constants, {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(),
                              Op.L: L.data_ptr()})
    torch.cuda.synchronize()
    out = {"O": O.cpu().numpy(), "L": L.cpu().numpy() / np.float32(1.44269504089)}
    _check_forward(desc, net, out, True, 1e-3)


BACKWARD_SHAPES = [(128, 128, 64), (256, 256, 128), (384, 256, 64), (200, 333, 128), (77, 129, 64), (300, 17, 80),
                   (129, 257, 72), (1, 1, 8), (512, 640, 96), (1024, 1024, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", BACKWARD_SHAPES)
def test_causal_backward_bf16(R, C, D):
    _backward(R, C, D, "bf16", seed=R + 3 * C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", BACKWARD_SHAPES[:6])
@pytest.mark.parametrize("mode", ["fp16", "reference"])
def test_causal_backward_fp16_and_reference_policy(R, C, D, mode):
    _backward(R, C, D, mode, seed=5 * R + C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode", [(256, 256, 256, "bf16"), (200, 333, 192, "reference"), (130, 64, 160, "fp16"),
                                        (64, 1000, 256, "bf16"), (512, 640, 256, "fp16")])
def test_causal_backward_wide_heads(R, C, D, mode):
    _backward(R, C, D, mode, seed=R + 5 * C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode", [(700, 900, 128, "bf16"), (900, 700, 64, "reference"), (2048, 2048, 128, "bf16"),
                                        (1000, 520, 72, "fp16"), (1024, 1024, 256, "bf16"), (640, 2048, 64, "bf16")])
def test_causal_backward_traversal_split(R, C, D, mode):
    """Split backward grids: ranges of the traversal axis wholly past the diagonal still write (zero) partials."""
    desc = _descriptor(R, C, D, mode)
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    for t in (KT.backwardQuery, KT.backwardKeyValue):
        assert mfa.AttentionKernel(desc.kernelDescriptor(t)).launchCount(constants) == 2, t
    _backward(R, C, D, mode, seed=R + C + D)


@pytest.mark.gpu
def test_causal_backward_large_grid_converts_dO_once():
    from tests.attention_harness import run_attention
    from tests.test_tcgen05_backward import _rel_rms
    H, R, C, D = 40, 300, 640, 64
    desc = _descriptor(R, C, D, "reference", batch=H)
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    assert mfa.AttentionKernel(desc.kernelDescriptor(KT.backwardKeyValue)).launchCount(constants) == 2
    nets = [Network(R, C, D, seed=300 + h, threads=8, causal=True).round_inputs(1, 2) for h in range(H)]
    inputs = {getattr(Op, k): np.stack([getattr(n, k) for n in nets]) for k in ("Q", "K", "V", "dO")}
    out = run_attention(desc, None, inputs=inputs)
    for h in (0, 17, H - 1):
        for name, expected in {"dV": nets[h].derivativeV(), "dK": nets[h].derivativeK(),
                               "dQ": nets[h].derivativeQ()}.items():
            rel = _rel_rms(out[name][h], expected)
            assert rel <= 3e-4, (name, h, rel)


@pytest.mark.gpu
@pytest.mark.parametrize("mask", [1, 6, 10, 15])
@pytest.mark.parametrize("R,C,D", [(136, 200, 64), (256, 384, 128), (200, 136, 256)])
def test_causal_transposed_operands(R, C, D, mask):
    """Transposed operands are staged row-major; the mask lives in the kernels."""
    t = tuple(bool(mask & (1 << i)) for i in range(4))
    mode = "bf16" if mask & 1 else ("reference" if mask % 4 == 2 else "fp16")
    _forward(R, C, D, mode, seed=mask + R, transpose=t)
    _backward(R, C, D, mode, seed=mask + R + 1, transpose=t)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode", [(160, 160, 35, "reference"), (257, 129, 77, "bf16"), (300, 300, 100, "bf16"),
                                        (64, 640, 3, "reference"), (150, 210, 133, "bf16")])
def test_causal_head_dimensions_not_multiples_of_8(R, C, D, mode):
    _forward(R, C, D, mode, seed=R + C + D)
    _backward(R, C, D, mode, seed=R + C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", [(64, 64, 32), (130, 70, 64), (77, 200, 48), (100, 100, 300), (90, 40, 300)])
def test_causal_simt_fp32(R, C, D):
    _forward(R, C, D, "fp32", seed=R + C + D)
    _backward(R, C, D, "fp32", seed=R + C + D + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_causal_batched_heads_equal_their_single_head_runs(mode):
    from tests.attention_harness import run_attention
    R, C, D, H = 300, 512, 64, 3
    nets = [_network(_descriptor(R, C, D, mode), seed=21 + h) for h in range(H)]
    inputs = {getattr(Op, k): np.stack([getattr(n, k) for n in nets]) for k in ("Q", "K", "V", "dO")}
    out = run_attention(_descriptor(R, C, D, mode, batch=H), None, inputs=inputs)
    tol = 2e-5 if mode == "fp32" else 5e-2
    for h, net in enumerate(nets):
        single = run_attention(_descriptor(R, C, D, mode), net)
        ref = {"O": net.inferenceAttention(), "dQ": net.derivativeQ(), "dK": net.derivativeK(), "dV": net.derivativeV()}
        for name in ("O", "L", "D", "dQ", "dK", "dV"):
            np.testing.assert_allclose(out[name][h], single[name], rtol=1e-5, atol=1e-5, err_msg=f"{name}[{h}]")
        for name, expected in ref.items():
            assert np.abs(out[name][h] - expected).max() <= tol, (name, h)


@pytest.mark.gpu
@pytest.mark.parametrize("batch,R,C,D,mode", [(1, 200, 333, 64, "bf16"), (19, 130, 70, 64, "fp16"),
                                              (40, 1024, 1024, 128, "bf16"), (3, 64, 48, 24, "fp32")])
def test_causal_run_host(batch, R, C, D, mode):
    """mfa_attention_run_host fetches its kernels from the descriptor-keyed cache: causal must reach them."""
    from tests.test_run_host import _host_run
    desc = _descriptor(R, C, D, mode, batch=batch)
    nets = [_network(_descriptor(R, C, D, mode), seed=100 + b) for b in range(batch)]
    # an unmasked run first puts the unmasked kernels into the cache
    _host_run(_descriptor(R, C, D, mode, batch=batch, causal=False), nets[:1] * batch, list(KT), True)
    out = _host_run(desc, nets, list(KT), True)
    tol = 2e-5 if mode == "fp32" else 5e-2
    e = _empty_rows(R, C)
    for b in sorted({0, batch // 2, batch - 1}):
        n = nets[b]
        O, L = n.inferenceAttention(with_L=True)
        assert np.abs(out["O"][b] - O).max() <= tol
        assert np.isposinf(out["L"][b][:e]).all()
        assert np.abs(out["L"][b][e:] / np.float32(1.44269504089) - L[e:]).max() <= (2e-5 if mode == "fp32" else 7e-3)
        for name, expected in (("dV", n.derivativeV()), ("dK", n.derivativeK()), ("dQ", n.derivativeQ())):
            assert np.abs(out[name][b] - expected).max() <= tol, (name, b)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16", "reference", "fp32"])
@pytest.mark.parametrize("R,C,D", [(300, 17, 80), (130, 70, 256), (200, 64, 64)])
def test_causal_rows_without_a_visible_key_are_exact(R, C, D, mode):
    """R > C: O = 0, L = +inf, D = 0, dQ = 0 on the first R - C rows, and dK / dV are those of the problem without
    them (its last C rows, a square causal problem)."""
    from tests.test_tcgen05_backward import _rel_rms
    out, _ = _backward(R, C, D, mode, seed=R * C + D)
    e = R - C
    assert (out["O"][:e] == 0).all() and np.isposinf(out["L"][:e]).all()
    assert (out["D"][:e] == 0).all() and (out["dQ"][:e] == 0).all()
    net = _network(_descriptor(R, C, D, mode), seed=R * C + D)
    tail = Network(C, C, D, causal=True)
    tail.Q, tail.K, tail.V, tail.dO = net.Q[e:].copy(), net.K, net.V, net.dO[e:].copy()
    for name, expected in (("dK", tail.derivativeK()), ("dV", tail.derivativeV())):
        if mode == "fp32":
            assert np.abs(out[name] - expected).max() <= 2e-5, name
        else:
            bound = (2.5e-3 if mode == "bf16" else 3e-4) * (1.5 if C < 32 else 1.0)  # few terms per key, as in _backward
            assert _rel_rms(out[name], expected) <= bound, name


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,batch,t", [(4096, 4096, 128, 1, KT.forward), (300, 2000, 64, 2, KT.backwardQuery),
                                           (1000, 520, 72, 1, KT.backwardKeyValue)])
def test_causal_launch_count_is_what_encode_launches(R, C, D, batch, t):
    import torch
    from torch.profiler import ProfilerActivity, profile
    d = _descriptor(R, C, D, "bf16", batch=batch)
    c = mfa.FunctionConstantValues()
    d.setFunctionConstants(c)
    kernel = mfa.AttentionKernel(d.kernelDescriptor(t))
    assert kernel.sourceName().endswith("_causal")
    assert kernel.launchCount(c) == mfa.AttentionKernel(_descriptor(R, C, D, "bf16", batch=batch, causal=False)
                                                        .kernelDescriptor(t)).launchCount(c)
    torch.manual_seed(R + C)
    bufs = {}
    for op in (Op.Q, Op.K, Op.V, Op.O, Op.L, Op.D, Op.dO, Op.dV, Op.dK, Op.dQ):
        n = d.operandElements(op)
        bufs[op] = (torch.randn(n, device="cuda") if d.memoryPrecisions[op] == P.FP32 else
                    torch.randn(n, device="cuda").to(torch.bfloat16))
    bufs[Op.L].zero_()
    bufs[Op.D].zero_()
    ptrs = {op: b.data_ptr() for op, b in bufs.items()}
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
    assert len(launched) == kernel.launchCount(c), launched


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,mode", [(4096, 4096, 128, "bf16"), (640, 2048, 64, "bf16"), (300, 17, 80, "reference"),
                                        (1000, 520, 72, "fp16"), (130, 70, 256, "bf16"), (90, 40, 300, "fp32")])
def test_causal_results_are_deterministic(R, C, D, mode):
    """The kernels use no atomics and every split partial is written, fully masked or not: two runs of the same problem
    (forward, dQ, dK/dV; split grids, rows with no visible key, the staged and FP32 paths) are bitwise identical."""
    from tests.attention_harness import run_attention
    desc = _descriptor(R, C, D, mode)
    net = _network(desc, seed=R + C)
    first = run_attention(desc, net, return_raw=True)
    second = run_attention(desc, net, return_raw=True)
    for name, a in first.items():
        assert a.tobytes() == second[name].tobytes(), name
