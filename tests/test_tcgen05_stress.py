"""Seeded random shapes through the tensor-core family (forward and backward for D <= 256): ragged R and C,
every D % 8 == 0, the three 16-bit operand policies, small batches -- chosen so that the split paths (forward split-KV,
backward traversal split, ragged last ranges), the D <= 256 kernel's masked tails and the reference-policy dO conversion
all get exercised against the CPU oracle; a second list draws random transpose states (sequence lengths rounded to
multiples of 8, which the transposed TMA views need) for the staged (transposed) path.  Tolerances as in test_tcgen05_forward.py / test_tcgen05_backward.py."""
import numpy as np
import pytest


def _cases(count, seed, transposed=False):
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(count):
        R = int(rng.integers(1, 1400))
        C = int(rng.integers(1, 1400))
        D = int(rng.integers(1, 33)) * 8                      # 8 .. 256
        policy = ("bf16", "fp16", "reference")[int(rng.integers(0, 3))]
        lowMid = bool(rng.integers(0, 2))
        batch = int(rng.integers(1, 4))
        transpose = (False,) * 4
        if transposed:
            mask = int(rng.integers(1, 16))
            transpose = tuple(bool(mask & (1 << i)) for i in range(4))
            R, C = max(8, R // 8 * 8), max(8, C // 8 * 8)
        cases.append((R, C, D, policy, lowMid, batch, transpose))
    return cases


CASES = _cases(28, seed=20260923) + _cases(20, seed=7, transposed=True)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)))
def test_random_shape(case):
    import mfa_b200 as mfa
    import oracle
    from tests.attention_harness import run_attention, check

    R, C, D, policy, lowMid, batch, transpose = CASES[case]
    KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.lowPrecisionIntermediates = lowMid
    if policy != "reference":
        desc.inputPrecisionOverride = P.BF16 if policy == "bf16" else P.FP16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = transpose
    desc.batchCount = batch
    backward = True
    types = list(KT)
    for t in types:
        assert desc.kernelDescriptor(t).backend == mfa.Backend.tcgen05, t
    prec = desc.memoryPrecisions
    nets = [oracle.Network(R, C, D, seed=1000 * case + b, threads=8).round_inputs(int(prec[Op.Q]), int(prec[Op.dO]))
            for b in range(batch)]
    inputs = {getattr(Op, k): np.stack([getattr(n, k) for n in nets]) if batch > 1 else getattr(nets[0], k)
              for k in ("Q", "K", "V", "dO")}
    out = run_attention(desc, None, inputs=inputs, types=types)

    bf16 = policy == "bf16"

    def rel_rms(a, b):
        denom = float(np.sqrt(np.mean(b ** 2)))
        err = float(np.sqrt(np.mean((a - b) ** 2)))
        return err / denom if denom > 1e-12 else err

    for b, n in enumerate(nets):
        pick = (lambda a: a[b]) if batch > 1 else (lambda a: a)
        O, L = n.inferenceAttention(with_L=True)
        assert rel_rms(pick(out["O"]), O) <= (2e-3 if bf16 else 1e-3), ("O", b)
        check(L, pick(out["L"]), 7e-3 if lowMid else 1e-3, "L")
        if not backward:
            continue
        check(n.createDTerms(), pick(out["D"]), 1e-1 if lowMid else 2e-2, "D")
        bound = 4e-3 if bf16 else 1.5e-3
        if lowMid:
            bound = max(bound, 6e-3)   # L read back from FP16, D from BF16
        for name, expected in (("dV", n.derivativeV()), ("dK", n.derivativeK()), ("dQ", n.derivativeQ())):
            check(expected, pick(out[name]), 5e-2, name)
            assert rel_rms(pick(out[name]), expected) <= bound, (name, b)
