"""O, L, D, dQ, dK and dV of every tensor-core backward kernel (the dQ and dK/dV kernels of kernels/wgmma_attention.cu)
on seeded inputs, for comparing two builds of the library output for output, and kernel time for kernel time.

    MFA_B200_LIBRARY=/path/to/old/libmfa_b200.so python scripts/ab_wgmma_backward_outputs.py --out DIR_A [--time]
    python scripts/ab_wgmma_backward_outputs.py --out DIR_B [--time]
    python scripts/ab_wgmma_backward_outputs.py --compare DIR_A DIR_B    # exit status 1 unless every array is bitwise equal

CASES reach all 108 backward entry functions: fixed-length and packed calls, each causal, not causal and with a window
(the window kernels have no causal template parameter: their band carries the mask), at D = 64, 120 and 256 (DCH 1, 2,
4), in BF16, FP16 and FP16 with BF16 dO.  They rotate over G = 1 and 4 and 16-bit intermediates.  Two more cases cover
the launcher's other paths: a fixed call of one head and long sequences, whose dQ and dK/dV grids are split and summed
by sum_splits, and an FP16 + BF16-dO call whose dK/dV grid is more than one wave, so that dO is converted in a pass of
its own first.  The calls go through the test suites' runners, with NaN output sentinels, and each of their kernels
must run on Backend.tcgen05; the machinery is that of ab_simt_outputs.py.  The entry functions listed per case are
derived here from the case at the small sizes by the launcher's rules; the library reports only each kernel's backend
and launch count.

--time runs the same cases at a user's sizes instead (fixed R = C = 2048 with 16 heads; packed: 8 sequences of 1-2048
tokens with 16 heads; the two cases above at their own sizes) and records, per case and kernel type, the median
CUDA-event time of 20 launches after 3 warm-up launches.  It saves no arrays but a SHA-256 digest of each, which
--compare checks too."""
import contextlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts import ab_simt_outputs  # noqa: E402

SM_COUNT = 132   # the H100 SXM's SMs: the dO conversion pass runs when a dK/dV grid is larger


def _cases():
    """name: (form, D, mode, causal, G, 16-bit intermediates, window (left, right) or None, (H, R, C) or None)"""
    cases = {}
    i = 0
    for D in (64, 120, 256):
        for mode in ("bf16", "fp16", "reference"):
            for form in ("fixed", "packed"):
                for kind in ("causal", "plain", "window"):
                    window = ((63, 0), (30, 70), (100, 0))[i // 3 % 3] if kind == "window" else None
                    causal = kind == "causal" or (window is not None and window[1] == 0)
                    name = f"{form}_{kind}_d{D}_{mode}"
                    cases[name] = (form, D, mode, causal, (1, 4)[i % 2], i % 5 == 0, window, None)
                    i += 1
    cases["split_fixed_d128_bf16"] = ("fixed", 128, "bf16", False, 1, False, None, (1, 4096, 4096))
    cases["convert_first_fixed_d64_reference"] = ("fixed", 64, "reference", True, 1, False, None, (16, 2048, 2048))
    return cases


CASES = _cases()


def instantiations(case):
    """the backward entry functions a case launches at the small sizes"""
    form, D, mode, causal, G, _, window, shape = case
    dch = next(n for n in (1, 2, 4) if 64 * n >= D)
    bf16 = mode == "bf16"
    # CTAs of the dK/dV grid: key tiles of 128 rows (64 at D > 128) x K/V heads x sequences
    if shape is not None:
        H, C, count = shape[0], shape[2], 1
    elif form == "fixed":
        H, C, count = 4, 333, 1
    else:
        H, C, count = 4, max(ab_simt_outputs.SMALL[1]), len(ab_simt_outputs.SMALL[1])
    kv_ctas = -(-C // (64 if D > 128 else 128)) * H // G * count
    names = []
    for kind in ("query", "key_value"):
        convert = mode == "reference" and not (kind == "key_value" and kv_ctas > SM_COUNT)
        args = f"{dch}, {str(bf16).lower()}, {str(convert).lower()}"
        if window is not None:
            names.append(f"band_backward_{kind}{'_packed' if form == 'packed' else ''}_wgmma<{args}>")
        else:
            prefix = "attention" if form == "fixed" else "packed"
            names.append(f"{prefix}_backward_{kind}_wgmma<{args}, {str(causal).lower()}>")
    return names


assert len({f for case in CASES.values() for f in instantiations(case)}) == 108


def run_case(mfa, torch, seed, timed, form, D, mode, causal, G, lowMid, window, shape):
    """{output name: array} of one case, through the runner of its form"""
    from tests.test_window import windowed
    window_block = windowed(window) if window is not None else contextlib.nullcontext()
    if form == "fixed":
        from tests.test_kv_group import _descriptor, _inputs, run
        if shape is not None:
            H, R, C = shape
        else:
            H, (R, C) = (16, (2048, 2048)) if timed else (4, (200, 333) if seed % 2 else (333, 200))
        desc = _descriptor(R, C, D, mode, batch=H, causal=causal, lowMid=lowMid)
        x = _inputs(desc, G, seed)
        with window_block:
            return run(desc, G, x, raw=True)
    from tests.test_varlen import _descriptor, _inputs, _offsets, run_packed
    H = 16 if timed else 4
    rq, rk = ab_simt_outputs.TIMED if timed else ab_simt_outputs.SMALL
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 9, ko[-1] + 5   # rows past the table's end keep their sentinels
    desc = _descriptor(T, Tk, D, mode, H, causal, lowMid=lowMid)
    x = _inputs(desc, G, T, Tk, seed)
    with window_block:
        return run_packed(desc, G, x, qo, ko)


if __name__ == "__main__":
    ab_simt_outputs.main(cases=CASES, run=run_case, functions=instantiations, backend="tcgen05")
