"""The wgmma pipeline: what ptxas made of the tensor-core kernels, and forward shapes at the edges of the key loop.

The K steps of a wgmma product only run back to back if ptxas keeps the wgmma pipeline asynchronous: a function call
anywhere in a kernel (a device printf, say) makes it serialize every wgmma of that kernel (warning C7510), and a spill
or a stack frame would put local memory traffic into the loops.  The GPU tests run the forward at 1 to 5 key blocks per
CTA, causal tiles and split ranges that see no key, and split ranges of an odd number of blocks, twice each."""
import os
import re

import numpy as np
import pytest

import mfa_b200 as mfa

KT, Op = mfa.AttentionKernelType, mfa.AttentionOperand
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "metal-flash-attention_b200", "_build", "kernels", "wgmma_attention.o.ptxas.log")


def _ptxas_report():
    """{kernel (mangled name): (stack frame bytes, spill store bytes, spill load bytes)} and the log's text."""
    assert os.path.exists(PTXAS_LOG), f"{PTXAS_LOG} is missing: build() writes it when it compiles the library"
    with open(PTXAS_LOG) as f:
        text = f.read()
    report, function = {}, None
    for line in text.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            function = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and function is not None:
            report[function] = tuple(int(x) for x in m.groups())
            function = None
    return report, text


def test_ptxas_serializes_no_wgmma():
    _, text = _ptxas_report()
    serialized = sorted(set(re.findall(r"C7510.*?function '(\S+)'", text)))
    assert not serialized, "ptxas serialized the wgmma pipeline of:\n" + "\n".join(serialized)


def test_tensor_core_kernels_have_no_spills_and_no_stack_frame():
    report, _ = _ptxas_report()
    # every entry function (mangled "<name>_wgmmaI<template arguments>"): the forward's call forms, and the dQ and dK/dV
    # kernels, of which several sit within a few registers of the limit
    kernels = {name: r for name, r in report.items() if re.search(r"_wgmmaI", name)}
    # 3 head-dimension chunk counts x each form's type / mask / dO-conversion instantiations
    assert len(kernels) == 216, sorted(kernels)
    assert len([name for name in kernels if "backward" in name]) == 108, sorted(kernels)
    bad = {name: r for name, r in kernels.items() if r != (0, 0, 0)}
    assert not bad, "stack frame / spill stores / spill loads (bytes): " + repr(bad)


# ------------------------------------------------------------------------------------------------ GPU
def _run_twice(R, C, D, causal, split, seed):
    """The bf16 forward of one seeded problem with the given split policy, run twice on fresh NaN-filled outputs: both
    runs must be bitwise identical, and match the oracle.  Returns the launch count (2 = split grid + merge)."""
    import torch
    from tests.test_causal import _check_forward, _descriptor, _network
    desc = _descriptor(R, C, D, "bf16", causal=causal)
    kd = desc.kernelDescriptor(KT.forward)
    assert kd.backend == mfa.Backend.tcgen05
    kd.splitPolicy = split
    kernel = mfa.AttentionKernel(kd)
    constants = mfa.FunctionConstantValues()
    desc.setFunctionConstants(constants)
    net = _network(desc, seed, causal=causal)
    q, k, v = (torch.from_numpy(np.asarray(x, np.float32)).to(torch.bfloat16).cuda() for x in (net.Q, net.K, net.V))
    runs = []
    for _ in range(2):
        O = torch.full((R, D), float("nan"), device="cuda")
        L = torch.full((R,), float("nan"), device="cuda")
        kernel.encode(constants, {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(),
                                  Op.L: L.data_ptr()})
        torch.cuda.synchronize()
        runs.append((O.cpu().numpy(), L.cpu().numpy()))
    assert runs[0][0].tobytes() == runs[1][0].tobytes() and runs[0][1].tobytes() == runs[1][1].tobytes()
    out = {"O": runs[0][0], "L": runs[0][1] / np.float32(1.44269504089)}
    if causal:
        _check_forward(desc, net, out, True, 1e-3)
    else:   # (_check_forward expects the R - C rows of the causal mask that see no key)
        from tests.attention_harness import check
        from tests.test_tcgen05_forward import check_O
        O, L = net.inferenceAttention(with_L=True)
        check_O(O, out["O"], net.V, True)
        check(L, out["L"], 1e-3, "L")
    return kernel.launchCount(constants)


NO_SPLIT = (0, 1)

# Every CTA sees 1, 2, 3, 4 and 5 key blocks (128 keys at D <= 128, 64 at D = 256), ragged or whole, unsplit
KEY_BLOCK_SHAPES = [
    (160, 100, 64), (160, 250, 64), (160, 384, 64), (160, 500, 64), (160, 640, 64),
    (136, 128, 128), (136, 200, 128), (136, 300, 128), (136, 512, 128), (136, 600, 128),
    (130, 40, 256), (130, 128, 256), (130, 150, 256), (130, 256, 256), (130, 300, 256),
]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D", KEY_BLOCK_SHAPES)
def test_forward_key_blocks_per_cta(R, C, D):
    assert _run_twice(R, C, D, causal=False, split=NO_SPLIT, seed=R + C + D) == 1


# Causal, R > C: whole query tiles see no key (blocks = 0), the others see 1, 2, ... blocks; split, whole key ranges of a
# tile lie past the diagonal
@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,split,launches", [
    (600, 300, 128, NO_SPLIT, 1), (600, 300, 128, (1, 4), 2),
    (700, 450, 64, NO_SPLIT, 1), (700, 450, 64, (1, 4), 2),
    (520, 200, 256, NO_SPLIT, 1), (520, 200, 256, (1, 4), 2),
])
def test_causal_forward_with_empty_tiles(R, C, D, split, launches):
    assert _run_twice(R, C, D, causal=True, split=split, seed=3 * R + C + D) == launches


# Split grids with an odd number of key blocks per split range: 2 ranges of 3 or 5 blocks
@pytest.mark.gpu
@pytest.mark.parametrize("R,C,D,split", [(256, 768, 128, (3, 2)), (200, 1280, 64, (5, 2)), (256, 384, 256, (3, 2)),
                                         (300, 700, 128, (3, 2))])
@pytest.mark.parametrize("causal", [False, True], ids=["unmasked", "causal"])
def test_forward_split_with_odd_blocks_per_range(R, C, D, split, causal):
    assert _run_twice(R, C, D, causal=causal, split=split, seed=R + 5 * C + D) == 2
