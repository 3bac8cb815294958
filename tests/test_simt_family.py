"""The SIMT family (kernels/simt_attention.cu): its ptxas report.

Every SIMT kernel runs one 256-thread CTA per SM at 156-255 registers, so a change to a shared body can push an
instantiation into spilling.  The report must list all 52 entry functions, and none may have a stack frame or spill
beyond the two dK/dV kernels that spilled before the bodies were shared, which may not spill more than they did then."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "metal-flash-attention_b200", "_build", "kernels", "simt_attention.o.ptxas.log")

# (kernel, NCH, Layout or None): fixed, packed (_varlen) and paged forwards, and the window (band) kernels per Layout
# (0 fixed, 1 packed, 2 paged); dK/dV stops at 4 chunks and slices wider heads
ENTRIES = (
    {(k, n, None) for k in ("simt_forward_kernel", "simt_forward_kernel_varlen", "simt_forward_kernel_paged",
                            "simt_backward_query_kernel", "simt_backward_query_kernel_varlen") for n in (1, 2, 4, 8)}
    | {("simt_band_forward_kernel", n, lay) for n in (1, 2, 4, 8) for lay in (0, 1, 2)}
    | {("simt_band_backward_query_kernel", n, lay) for n in (1, 2, 4, 8) for lay in (0, 1)}
    | {(k, n, None) for k in ("simt_backward_key_value_kernel", "simt_backward_key_value_kernel_varlen") for n in (1, 2, 4)}
    | {("simt_band_backward_key_value_kernel", n, lay) for n in (1, 2, 4) for lay in (0, 1)}
)
# (stack frame, spill stores, spill loads) in bytes, at most: what CUDA 12.9 made of these two kernels at the parent of
# the merge.  Since the merge the fixed one has no stack frame and no spills; the packed band one is unchanged.
SPILL_BUDGET = {
    ("simt_backward_key_value_kernel", 4, None): (8, 4, 8),
    ("simt_band_backward_key_value_kernel", 4, 1): (32, 32, 64),
}


def entry(mangled):
    """(kernel, NCH, Layout or None) of a mangled mfa::simt kernel name"""
    m = re.fullmatch(r"_ZN3mfa4simt\d+(\w+?)ILi(\d)E(?:LNS0_6LayoutE(\d)E)?EEv\w*", mangled)
    assert m, mangled
    return m.group(1), int(m.group(2)), None if m.group(3) is None else int(m.group(3))


def test_ptxas_simt_kernels_have_no_new_spills_and_no_new_stack_frames():
    assert os.path.exists(LOG), f"{LOG} is missing: build() writes it when it compiles the library"
    report, function = {}, None
    for line in open(LOG).read().splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            function = entry(m.group(1))
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and function is not None:
            report[function] = tuple(int(x) for x in m.groups())
            function = None
    assert len(ENTRIES) == 52
    assert set(report) == ENTRIES, sorted(set(report) ^ ENTRIES)
    over = {f: r for f, r in report.items()
            if any(got > limit for got, limit in zip(r, SPILL_BUDGET.get(f, (0, 0, 0))))}
    assert not over, over
