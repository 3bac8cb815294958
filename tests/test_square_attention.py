"""The reference's SquareAttentionTest.testCorrectness (Tests/FlashAttentionTests/Attention/
SquareAttentionTest.swift:5-26 -> validateProblemSize :214-555) against the sm_90a kernels through the
C ABI: the same 20 (N, D) shapes, FP32 everywhere, forward + dQ + dK/dV, absolute tolerance 2e-5 on
O, L, D, dV, dK, dQ (:547-554).  Inputs are seeded (the reference's are not); failures assert (the
reference only prints)."""
import numpy as np
import pytest

REFERENCE_SHAPES = [
    (10, 3), (10, 80), (8, 2), (9, 2), (23, 2), (24, 2), (25, 2), (192, 77), (192, 80), (93, 32),
    (99, 35), (64, 32), (64, 34), (64, 36), (64, 40), (32, 64), (4, 1), (4, 2), (384, 95), (777, 199),
]


def validateProblemSize(sequenceDimension, headDimension, seed=0):
    import mfa_b200 as mfa
    from oracle import Network
    from tests.attention_harness import run_attention, oracle_outputs, check

    network = Network(sequenceDimension, sequenceDimension, headDimension, seed=seed)

    attentionDesc = mfa.AttentionDescriptor()
    attentionDesc.lowPrecisionInputs = False
    attentionDesc.lowPrecisionIntermediates = False
    attentionDesc.matrixDimensions = (sequenceDimension, sequenceDimension, headDimension)
    attentionDesc.transposeState = (False, False, False, False)

    result = run_attention(attentionDesc, network)
    expected = oracle_outputs(network)
    # FP32 path: 2e-5 on everything (SquareAttentionTest.swift:547-554)
    for name in ("O", "L", "D", "dV", "dK", "dQ"):
        check(expected[name], result[name], 2e-5, name)


@pytest.mark.gpu
@pytest.mark.parametrize("sequenceDimension,headDimension", REFERENCE_SHAPES)
def test_correctness(sequenceDimension, headDimension):
    validateProblemSize(sequenceDimension, headDimension, seed=sequenceDimension * 1000 + headDimension)


@pytest.mark.gpu
def test_config1_plumbing_fp32_n128_d64():
    """BASELINE.json configs[0]: single-head forward N=128 D=64 FP32 (the reference's CPU-runnable case)."""
    validateProblemSize(128, 64, seed=1)


@pytest.mark.gpu
def test_large_head_dimension_and_batch():
    """D up to 512 (accumulator slicing in the dK/dV kernel) and the batch extension."""
    import mfa_b200 as mfa
    from oracle import Network
    from tests.attention_harness import run_attention, oracle_outputs, check

    validateProblemSize(70, 300, seed=5)
    validateProblemSize(40, 512, seed=6)
    nets = [Network(50, 37, 24, seed=s) for s in (1, 2, 3)]
    desc = mfa.AttentionDescriptor()
    desc.matrixDimensions = (50, 37, 24)
    desc.transposeState = (False, True, False, True)
    desc.batchCount = 3
    inputs = {getattr(mfa.AttentionOperand, k): np.stack([getattr(n, k) for n in nets]) for k in ("Q", "K", "V", "dO")}
    result = run_attention(desc, None, inputs=inputs)
    for b, n in enumerate(nets):
        expected = oracle_outputs(n)
        for name in ("O", "L", "D", "dV", "dK", "dQ"):
            check(expected[name], result[name][b], 2e-5, f"{name}[batch {b}]")
