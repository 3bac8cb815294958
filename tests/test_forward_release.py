"""The unmasked fixed-length forward, whose key loop frees ring stages through mbarriers instead of a CTA-wide barrier:
the two warpgroups of a CTA drift apart, and thread 0 refills a stage only after both have released it.

Ragged and whole tile counts, split key ranges of an odd number of blocks and grouped K/V, at every head-dimension
kernel.  Each case runs twice on fresh NaN-poisoned outputs whose tails must survive, bitwise equal, and is checked
against the float64 reference of tests/causal_oracle.attention_f64, with grouped K/V where G > 1."""
import numpy as np
import pytest

import mfa_b200 as mfa
from tests.test_kv_group import _descriptor, _inputs, reference, run

KT, Op = mfa.AttentionKernelType, mfa.AttentionOperand
NO_SPLIT = (0, 1)


def _run_twice(R, C, D, B=1, G=1, split=NO_SPLIT, seed=0):
    """O and L of the bf16 forward, twice, bitwise equal and within the forward suites' tolerances of the reference.
    Returns the launch count (2 = split grid + merge)."""
    from tests.attention_harness import check
    from tests.test_tcgen05_forward import check_O
    desc = _descriptor(R, C, D, "bf16", batch=B)
    kd = desc.kernelDescriptor(KT.forward)
    assert kd.backend == mfa.Backend.tcgen05
    inputs = _inputs(desc, G, seed)

    def edit(kd):
        kd.splitPolicy = split

    runs = [run(desc, G, inputs, types=(KT.forward,), edit=edit, raw=True) for _ in range(2)]
    for name in ("O", "L"):
        assert runs[0][name].tobytes() == runs[1][name].tobytes(), f"{name} differs between two runs"
    ref = reference(inputs, G, causal=False)
    check_O(ref["O"], runs[0]["O"], inputs[Op.V], True)
    check(ref["L"], runs[0]["L"] / np.float32(1.44269504089), 1e-3, "L")
    c = mfa.FunctionConstantValues()
    desc.setFunctionConstants(c)
    c.kvGroup = G
    kd.splitPolicy = split
    return mfa.AttentionKernel(kd).launchCount(c)


# 1 to 5 query tiles of 128 rows, ragged or whole, at every head-dimension kernel
@pytest.mark.gpu
@pytest.mark.parametrize("R", [100, 128, 136, 300, 392, 640])
@pytest.mark.parametrize("C,D", [(333, 64), (300, 128), (200, 256)])
def test_tile_counts(R, C, D):
    assert _run_twice(R, C, D, B=3, seed=R + C + D) == 1


# Split key ranges of an odd number of blocks (blockIdx.z), over odd and even tile counts
@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,split", [(300, 768, 128, (3, 2)), (136, 1280, 64, (5, 2)), (100, 384, 256, (3, 2)),
                                         (392, 700, 128, (3, 2))])
def test_split_ranges(R, C, D, split):
    assert _run_twice(R, C, D, B=1, split=split, seed=R + 5 * C + D) == 2


# Grouped K/V: four query heads per K/V head
@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", [(300, 257, 128), (136, 500, 64), (130, 150, 256)])
def test_grouped_kv(R, C, D):
    assert _run_twice(R, C, D, B=8, G=4, seed=R + C + D + 4) == 1
