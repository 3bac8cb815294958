"""Parity of the tensor-core backward kernels (dQ and dK/dV, TMA + wgmma) with the CPU oracle, on inputs
rounded to the kernels' 16-bit memory format.  Forward runs first (it produces O and L), then backwardQuery (writes
D and dQ), then backwardKeyValue -- the reference's order (SquareAttentionTest.swift:355-368).

Stated tolerances: the reference's mixed-precision bars (D 1e-1, gradients 5e-2, RectangularAttentionTest.swift:
459-464) and, tighter, relative RMS error of every gradient <= 2.5e-3 for BF16 / 3e-4 for FP16: the quantisation floor
of the 16-bit MMA operands P and dS (2^-s / sqrt(6) per rounded operand, s = 8 / 11 significant bits: 1.6e-3 / 2.0e-4;
small shapes scatter a little above the asymptotic value)."""
import numpy as np
import pytest


def _rel_rms(actual, expected):
    denom = float(np.sqrt(np.mean(expected ** 2)))
    err = float(np.sqrt(np.mean((actual - expected) ** 2)))
    return err / denom if denom > 1e-12 else err   # e.g. C == 1: dS == 0, so dK == dQ == 0 exactly


def _run(R, C, D, bf16, seed, lowMid=False, referencePolicy=False, transpose=(False, False, False, False)):
    import mfa_b200 as mfa
    import oracle
    from tests.attention_harness import run_attention, oracle_outputs, check

    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.lowPrecisionIntermediates = lowMid
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = tuple(transpose)
    if referencePolicy:
        # the reference's own policy: FP16 Q, K, V and BF16 dO (AttentionDescriptor+Precisions.swift:13-23); the
        # kernels rewrite the staged dO tiles as FP16 on chip (wgmma cannot mix FP16 and BF16 operands)
        assert not bf16
        prec = desc.memoryPrecisions
        assert prec[mfa.AttentionOperand.Q] == mfa.GEMMOperandPrecision.FP16
        assert prec[mfa.AttentionOperand.dO] == mfa.GEMMOperandPrecision.BF16
    else:
        desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16 if bf16 else mfa.GEMMOperandPrecision.FP16
    for t in mfa.AttentionKernelType:
        assert desc.kernelDescriptor(t).backend == mfa.Backend.tcgen05, t
    net = oracle.Network(R, C, D, seed=seed, threads=8)
    prec = desc.memoryPrecisions
    net.round_inputs(int(prec[mfa.AttentionOperand.Q]), int(prec[mfa.AttentionOperand.dO]))
    out = run_attention(desc, net)
    ref = oracle_outputs(net)
    check(ref["D"], out["D"], 1e-1 if lowMid else 2e-2, "D")
    bound = 2.5e-3 if bf16 else 3e-4
    if min(R, C, D) < 16:
        bound *= 1.5   # a handful of terms per output element: the error does not average down to the asymptotic floor
    if lowMid and not bf16:
        bound = 2.5e-3   # L read back from FP16 (|L| ~ 8: half an ulp = 2^-8 in log2 units -> P off by up to 0.27 %)
    for name in ("dV", "dK", "dQ"):
        check(ref[name], out[name], 5e-2, name)
        rel = _rel_rms(out[name], ref[name])
        assert rel <= bound, f"{name}: relative RMS error {rel:.3e} > {bound}"
    return out, ref


SHAPES = [(128, 128, 64), (256, 256, 128), (384, 256, 64), (200, 333, 128), (77, 129, 64), (300, 17, 80),
          (129, 257, 72), (1, 1, 8), (512, 640, 96), (1024, 1024, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", SHAPES)
def test_backward_bf16_matches_oracle(R, C, D):
    _run(R, C, D, True, seed=R + 3 * C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", SHAPES[:6])
def test_backward_fp16_matches_oracle(R, C, D):
    _run(R, C, D, False, seed=5 * R + C + D)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,bf16,referencePolicy", [(700, 900, 128, True, False), (900, 700, 64, False, True),
                                                        (2048, 2048, 128, True, False), (1000, 520, 72, False, False)])
def test_backward_traversal_split_small_grids(R, C, D, bf16, referencePolicy):
    """Few CTAs for 132 SMs: the traversal axis (keys for dQ, queries for dK/dV) is cut into ranges handled by separate
    CTAs whose partial accumulators a sum kernel adds up; ragged last ranges, ragged last blocks."""
    import mfa_b200 as mfa
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    if not referencePolicy:
        desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16 if bf16 else mfa.GEMMOperandPrecision.FP16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = (False, False, False, False)
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    for t in (mfa.AttentionKernelType.backwardQuery, mfa.AttentionKernelType.backwardKeyValue):
        assert mfa.AttentionKernel(desc.kernelDescriptor(t)).launchCount(constants) == 2, t
    _run(R, C, D, bf16, seed=R + C + D, referencePolicy=referencePolicy)


@pytest.mark.gpu
def test_backward_low_precision_intermediates_bf16():
    """L stored FP16, D stored BF16 (AttentionDescriptor+Precisions.swift:81-87) and read back by dK/dV."""
    _run(256, 384, 64, True, seed=4, lowMid=True)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", [(128, 128, 64), (256, 256, 128), (200, 333, 128), (77, 129, 64), (300, 17, 80),
                                   (129, 257, 72), (1, 1, 8), (512, 640, 96), (640, 1024, 128)])
@pytest.mark.parametrize("lowMid", [False, True])
def test_backward_reference_policy_fp16_inputs_bf16_dO(R, C, D, lowMid):
    """The reference's unmodified low-precision descriptor (FP16 Q/K/V, BF16 dO; with lowPrecisionIntermediates also
    FP16 L and BF16 D) on the tensor-core kernels."""
    _run(R, C, D, False, seed=7 * R + C + D, lowMid=lowMid, referencePolicy=True)


@pytest.mark.gpu
def test_config3_fwd_bwd_n2048_d64():
    """BASELINE.json configs[2]: forward + backward (dQ, dK/dV) N=2048 D=64 on one H100 through the tensor-core family:
    the reference's policy (FP16 Q/K/V + BF16 dO, as the reference would run "fp16"), all-FP16 and all-BF16."""
    _run(2048, 2048, 64, False, seed=2, referencePolicy=True)
    _run(2048, 2048, 64, False, seed=0)
    _run(2048, 2048, 64, True, seed=1)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 128])
def test_table_split_policies_match_the_oracle(D):
    """The parameter table's small-grid split policy decides how the three kernels cut their traversal axis: every
    policy must give the same answers.  Shapes: a grid that is split (one head, 1024 x 1536) under two split policies,
    and ragged edges with the reference's precision policy."""
    import mfa_b200 as mfa
    KT = mfa.AttentionKernelType
    resident = {KT.forward: "Q, O", KT.backwardQuery: "Q, dO, dQ", KT.backwardKeyValue: "K, V, dV, dK"}
    par = {KT.forward: 128, KT.backwardQuery: 128, KT.backwardKeyValue: 128}
    trav = {KT.forward: 128, KT.backwardQuery: 64, KT.backwardKeyValue: 64}
    try:
        for policy in ((2, 8), (4, 3)):
            for t in KT:
                mfa.setParameterTable(t, f"| 128 | {par[t]} | {trav[t]} | 128 | {resident[t]} | {policy[0]} | {policy[1]} |\n")
            _run(1024, 1536, D, True, seed=D)
        _run(200, 333, D, False, seed=D + 1, referencePolicy=True)
    finally:
        for t in KT:
            mfa.setParameterTable(t, None)


@pytest.mark.gpu
def test_persistent_backward_many_items_per_cta():
    """D <= 64: both backward kernels are persistent (one CTA per SM walks the work items, barrier phases and ring stages
    carried across items, Q / dO resp. K / V double-buffered).  More items than SMs, ragged shapes, odd block counts, so
    that every phase pattern across an item boundary occurs."""
    import numpy as np
    import mfa_b200 as mfa
    import oracle
    from tests.attention_harness import run_attention, check
    Op = mfa.AttentionOperand
    for (H, R, C, D, bf16) in ((40, 640, 384, 64, True), (23, 300, 900, 40, False), (170, 128, 128, 64, True)):
        desc = mfa.AttentionDescriptor()
        desc.lowPrecisionInputs = True
        desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16 if bf16 else mfa.GEMMOperandPrecision.FP16
        desc.matrixDimensions = (R, C, D)
        desc.transposeState = (False, False, False, False)
        desc.batchCount = H
        rounding = oracle.BF16 if bf16 else oracle.FP16
        nets = [oracle.Network(R, C, D, seed=900 + h, threads=8).round_inputs(rounding) for h in range(H)]
        inputs = {getattr(Op, k): np.stack([getattr(n, k) for n in nets]) for k in ("Q", "K", "V", "dO")}
        out = run_attention(desc, None, inputs=inputs)
        for h in sorted({0, 1, H // 2, H - 2, H - 1}):
            ref = {"dV": nets[h].derivativeV(), "dK": nets[h].derivativeK(), "dQ": nets[h].derivativeQ()}
            for name, expected in ref.items():
                check(expected, out[name][h], 5e-2, f"{name}[{h}]")
                rel = _rel_rms(out[name][h], expected)
                assert rel <= (2.5e-3 if bf16 else 3e-4), (name, h, rel)
        assert all(np.isfinite(out[name]).all() for name in ("D", "dQ", "dK", "dV"))


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", [(160, 160, 35), (257, 129, 77), (384, 200, 95), (64, 640, 3), (300, 300, 100)])
@pytest.mark.parametrize("policy", ["reference", "bf16"])
def test_head_dimensions_that_are_not_multiples_of_8_run_on_the_tensor_cores(R, C, D, policy):
    """16-bit operands with D % 8 != 0 (the reference's own shapes: D = 35, 77, 95, ... SquareAttentionTest.swift:6-25) are
    staged with pad8(D) zero-padded columns and run on the tensor-core kernels (kernels/pad_head.cu); outputs come back
    un-padded, and nothing is written past them (the harness checks the poisoned tails)."""
    _run(R, C, D, policy == "bf16", seed=R + C + D, referencePolicy=policy == "reference")


@pytest.mark.gpu
def test_padded_forward_beyond_the_backward_kernels_reach():
    """D = 199 (reference shape list): forward on the tensor-core kernel for 128 < D <= 256 through padding to 200."""
    import mfa_b200 as mfa
    import oracle
    from tests.attention_harness import run_attention, check
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.matrixDimensions = (311, 190, 199)
    desc.transposeState = (False, False, False, False)
    assert desc.kernelDescriptor(mfa.AttentionKernelType.forward).backend == mfa.Backend.tcgen05
    net = oracle.Network(311, 190, 199, seed=8, threads=8).round_inputs(oracle.FP16)
    out = run_attention(desc, net, types=[mfa.AttentionKernelType.forward])
    O, L = net.inferenceAttention(with_L=True)
    check(O, out["O"], 2e-3, "O")
    check(L, out["L"], 1e-3, "L")
    assert _rel_rms(out["O"], O) <= 1e-3


# ---- wide heads (128 < D <= 256) and transposed (staged) operands ----
WIDE_SHAPES = [(256, 256, 256), (200, 333, 192), (77, 129, 136), (1, 1, 136), (512, 640, 256), (130, 64, 160),
               (64, 1000, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", WIDE_SHAPES)
@pytest.mark.parametrize("mode", ["bf16", "fp16", "reference"])
def test_backward_wide_heads_match_oracle(R, C, D, mode):
    """128 < D <= 256 on the tensor cores: 64-row tiles, dK / dV columns split over the two warpgroups."""
    _run(R, C, D, mode == "bf16", seed=R + 5 * C + D, referencePolicy=mode == "reference")


@pytest.mark.gpu
@pytest.mark.parametrize("mask", range(1, 16))
@pytest.mark.parametrize("R,C,D", [(136, 200, 64), (256, 384, 128), (200, 136, 256)])
def test_backward_transposed_operands_match_oracle(R, C, D, mask):
    """Every transpose state (Q, K, V, O; dO / dQ / dK / dV follow their primal, AttentionKernel.swift:189-195) through
    the tensor-core kernels (operands staged row-major first)."""
    t = tuple(bool(mask & (1 << i)) for i in range(4))
    bf16 = bool(mask & 1)
    _run(R, C, D, bf16, seed=mask + R, transpose=t, referencePolicy=(not bf16) and mask % 4 == 2)


@pytest.mark.gpu
def test_backward_transposed_low_precision_intermediates():
    _run(264, 392, 192, False, seed=11, lowMid=True, referencePolicy=True, transpose=(True, False, True, True))


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,transpose", [(1024, 1024, 256, (False,) * 4), (904, 712, 256, (True, True, False, True)),
                                             (2048, 2048, 128, (False, True, True, False))])
def test_backward_generic_traversal_split(R, C, D, transpose):
    """Few CTAs, wide heads and transposed operands: the traversal axis is split as for D <= 128, with one
    deterministic merge per kernel; transposed operands add one staging copy each."""
    import mfa_b200 as mfa
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = transpose
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    # a transposed operand is copied row-major before the kernel (an output: back after it); derived operands follow
    # their primal (dQ ~ Q, dK ~ K, dV ~ V, dO ~ O)
    t = dict(zip("QKVO", transpose))
    staged_q = 2 * t["Q"] + t["K"] + t["V"] + 2 * t["O"]     # Q, dQ, K, V, O, dO
    staged_kv = t["Q"] + 2 * t["K"] + 2 * t["V"] + t["O"]    # Q, K, dK, V, dV, dO
    # kernel + sum of the split partials (dK and dV in one pass at every D)
    assert mfa.AttentionKernel(desc.kernelDescriptor(mfa.AttentionKernelType.backwardQuery)).launchCount(constants) == (
        2 + staged_q)
    assert mfa.AttentionKernel(desc.kernelDescriptor(mfa.AttentionKernelType.backwardKeyValue)).launchCount(constants) == (
        2 + staged_kv)
    _run(R, C, D, True, seed=R + C, transpose=transpose)


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", [(150, 210, 133), (64, 64, 250)])
def test_backward_wide_head_not_multiple_of_8(R, C, D):
    """D % 8 != 0 beyond 128: staged with zero-padded columns, then the wide-head kernels."""
    _run(R, C, D, True, seed=D)


@pytest.mark.gpu
def test_backward_wide_heads_batched():
    """Several heads per launch through the generic kernels (work item -> (head, tile))."""
    import mfa_b200 as mfa
    import oracle
    from tests.attention_harness import run_attention, oracle_outputs
    R, C, D, H = 200, 264, 256, 5
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = (False, True, False, True)
    desc.batchCount = H
    nets = [oracle.Network(R, C, D, seed=40 + i, threads=8) for i in range(H)]
    prec = desc.memoryPrecisions
    for n in nets:
        n.round_inputs(int(prec[mfa.AttentionOperand.Q]), int(prec[mfa.AttentionOperand.dO]))
    inputs = {op: np.stack([getattr(n, op.name) for n in nets]) for op in
              (mfa.AttentionOperand.Q, mfa.AttentionOperand.K, mfa.AttentionOperand.V, mfa.AttentionOperand.dO)}
    out = run_attention(desc, None, inputs=inputs)
    for i, n in enumerate(nets):
        ref = oracle_outputs(n)
        for name in ("dQ", "dK", "dV"):
            rel = _rel_rms(out[name][i], ref[name])
            assert rel <= 2.5e-3, f"head {i} {name}: {rel:.3e}"


@pytest.mark.gpu
def test_reference_policy_large_grid_converts_dO_once():
    """FP16 Q/K/V beside BF16 dO with more key tiles than SMs: dK/dV converts dO in a pass of its own (one more launch)
    and runs the all-FP16 kernel; dQ keeps the in-kernel rewrite."""
    import mfa_b200 as mfa
    import oracle
    from tests.attention_harness import run_attention
    Op = mfa.AttentionOperand
    H, R, C, D = 40, 300, 640, 64
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = (False, False, False, False)
    desc.batchCount = H
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    assert mfa.AttentionKernel(desc.kernelDescriptor(mfa.AttentionKernelType.backwardKeyValue)).launchCount(constants) == 2
    assert mfa.AttentionKernel(desc.kernelDescriptor(mfa.AttentionKernelType.backwardQuery)).launchCount(constants) == 1
    nets = [oracle.Network(R, C, D, seed=300 + h, threads=8).round_inputs(oracle.FP16, oracle.BF16) for h in range(H)]
    inputs = {getattr(Op, k): np.stack([getattr(n, k) for n in nets]) for k in ("Q", "K", "V", "dO")}
    out = run_attention(desc, None, inputs=inputs)
    for h in (0, 17, H - 1):
        for name, expected in {"dV": nets[h].derivativeV(), "dK": nets[h].derivativeK(), "dQ": nets[h].derivativeQ()}.items():
            rel = _rel_rms(out[name][h], expected)
            assert rel <= 3e-4, (name, h, rel)
