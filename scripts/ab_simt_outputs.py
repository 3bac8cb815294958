"""O, L, D, dQ, dK and dV of every SIMT kernel (kernels/simt_attention.cu) on seeded inputs, for comparing two builds
of the library output for output, and kernel time for kernel time.

    MFA_B200_LIBRARY=/path/to/old/libmfa_b200.so python scripts/ab_simt_outputs.py --out DIR_A [--time]
    python scripts/ab_simt_outputs.py --out DIR_B [--time]
    python scripts/ab_simt_outputs.py --compare DIR_A DIR_B    # exit status 1 unless every array is bitwise equal

CASES reach all 52 SIMT entry functions: fixed-length, packed and paged calls (paged: the forward only), each with and
without a window, at D = 40, 128, 200 and 512 (NCH 1, 2, 4, 8; dK/dV 1, 2, 4 and 4 over two slices).  They rotate
over FP32, FP16, BF16 and the reference's FP16 Q/K/V with BF16 dO, causal or not, G = 1 and 4, 16-bit intermediates,
and aligned and unaligned transposes.  16-bit operands reach the SIMT family only at D > 256 or with transposes the
tensor cores cannot stage (D % 8 != 0), so the 16-bit cases at D <= 256 carry such transposes, and every case checks
that each of its kernels runs on Backend.simtFP32.  The calls go through the test suites' runners, with NaN output
sentinels: the outputs are saved in full, sentinels included.  Packed and paged calls have an empty query sequence and
an empty key sequence.  The entry functions listed per case (instantiations(), and the 52 they add up to) are derived
here from the form, D and window by the launchers' rules; they are not observed from the library, which reports only
each kernel's backend and launch count.

--time runs the same cases at a user's sizes instead (fixed R = C = 2048 with 16 heads; packed and paged: 8 sequences
of 1-2048 tokens) and records, per case and kernel type, the median CUDA-event time of 20 launches after 3 warm-up
launches.  It saves no arrays but a SHA-256 digest of each, which --compare checks too.  shapes.json records each
case's instantiations, backends and launch counts."""
import argparse
import contextlib
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (form, D, mode, causal, G, 16-bit intermediates, transposes (Q, K, V, O), window (left, right) or None)
T4, UNALIGNED = (True,) * 4, (False, True, True, False)
CASES = {
    "fixed_d40": ("fixed", 40, "fp32", True, 1, False, (True, False, True, False), None),
    "fixed_d127": ("fixed", 127, "fp16", False, 4, False, T4, None),
    "fixed_d200": ("fixed", 200, "fp32", True, 4, True, (False,) * 4, None),
    "fixed_d512": ("fixed", 512, "bf16", False, 1, False, (False,) * 4, None),
    "window_fixed_d40": ("fixed", 40, "fp32", True, 4, False, (False,) * 4, (63, 0)),
    "window_fixed_d128": ("fixed", 128, "fp32", False, 1, True, T4, (30, 70)),
    "window_fixed_d196": ("fixed", 196, "bf16", True, 4, False, UNALIGNED, (100, 0)),
    "window_fixed_d512": ("fixed", 512, "reference", False, 4, False, (False,) * 4, (200, 50)),
    "packed_d40": ("packed", 40, "fp32", True, 1, False, None, None),
    "packed_d128": ("packed", 128, "fp32", False, 4, True, None, None),
    "packed_d200": ("packed", 200, "fp32", True, 4, False, None, None),
    "packed_d512": ("packed", 512, "fp16", False, 1, False, None, None),
    "window_packed_d40": ("packed", 40, "fp32", False, 4, False, None, (20, 40)),
    "window_packed_d128": ("packed", 128, "fp32", True, 1, False, None, (63, 0)),
    "window_packed_d200": ("packed", 200, "fp32", False, 4, True, None, (-1, 3)),
    "window_packed_d512": ("packed", 512, "reference", True, 4, False, None, (100, 0)),
    "paged_d40": ("paged", 40, "fp32", True, 4, False, None, None),
    "paged_d128": ("paged", 128, "fp32", False, 1, False, None, None),
    "paged_d200": ("paged", 200, "fp32", True, 1, True, None, None),
    "paged_d512": ("paged", 512, "bf16", True, 4, False, None, None),
    "window_paged_d40": ("paged", 40, "fp32", True, 1, False, None, (100, 0)),
    "window_paged_d128": ("paged", 128, "fp32", False, 4, False, None, (30, 5)),
    "window_paged_d200": ("paged", 200, "fp32", False, 4, True, None, (0, 3)),
    "window_paged_d512": ("paged", 512, "fp16", True, 1, False, None, (63, 0)),
}
# query and key lengths of the packed and paged calls: Rs = 0 in the second sequence, Cs = 0 in the third
SMALL = ([70, 0, 130, 200, 1], [90, 50, 0, 100, 127])
TIMED = ([2048, 1, 1500, 64, 1024, 777, 300, 2000],) * 2
REPS, WARMUP = 20, 3


def instantiations(form, D, window):
    """the entry functions a case launches"""
    nch = next(n for n in (1, 2, 4, 8) if 64 * n >= D)
    layout = {"fixed": "kFixed", "packed": "kPacked", "paged": "kPaged"}[form]
    if window is not None:
        names = [f"simt_band_forward_kernel<{nch}, {layout}>", f"simt_band_backward_query_kernel<{nch}, {layout}>",
                 f"simt_band_backward_key_value_kernel<{min(nch, 4)}, {layout}>"]
    else:
        suffix = {"fixed": "", "packed": "_varlen", "paged": "_paged"}[form]
        names = [f"simt_forward_kernel{suffix}<{nch}>", f"simt_backward_query_kernel{suffix}<{nch}>",
                 f"simt_backward_key_value_kernel{suffix}<{min(nch, 4)}>"]
    return names[:1] if form == "paged" else names


assert len({f for c in CASES.values() for f in instantiations(c[0], c[1], c[7])}) == 52


@contextlib.contextmanager
def recorded(mfa, torch, record, timed):
    """Within the block, every AttentionKernel the runners create records its backend and launch count in
    record[kernel type], and with `timed` the median time of REPS launches of each encode after WARMUP."""
    plain = mfa.AttentionKernel

    class Recorded(plain):
        def __init__(self, descriptor, *args, **kwargs):
            super().__init__(descriptor, *args, **kwargs)
            self.kind = descriptor.type.name
            record.setdefault(self.kind, {})["backend"] = descriptor.backend.name

        def encode(self, constants, buffers, stream=0, **tables):
            entry = record[self.kind]
            entry["launches"] = self.launchCount(constants, **tables)
            if timed:
                for _ in range(WARMUP):
                    super().encode(constants, buffers, stream, **tables)
                events = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                          for _ in range(REPS)]
                for start, end in events:
                    start.record()
                    super().encode(constants, buffers, stream, **tables)
                    end.record()
                torch.cuda.synchronize()
                entry["ms"] = float(np.median([start.elapsed_time(end) for start, end in events]))
            super().encode(constants, buffers, stream, **tables)

    mfa.AttentionKernel = Recorded
    try:
        yield
    finally:
        mfa.AttentionKernel = plain


def run_case(mfa, torch, seed, timed, form, D, mode, causal, G, lowMid, transpose, window):
    """{output name: array} of one case, through the runner of its form"""
    from tests.test_window import windowed
    Op, H = mfa.AttentionOperand, 16 if timed else 4
    window_block = windowed(window) if window is not None else contextlib.nullcontext()
    if form == "fixed":
        from tests.test_kv_group import _descriptor, _inputs, run
        R, C = (2048, 2048) if timed else ((200, 333) if seed % 2 else (333, 200))
        desc = _descriptor(R, C, D, mode, batch=H, causal=causal, transpose=transpose, lowMid=lowMid)
        x = _inputs(desc, G, seed)
        with window_block:
            return run(desc, G, x, raw=True)
    from tests.test_varlen import _descriptor, _inputs, _offsets, run_packed
    rq, rk = TIMED if timed else SMALL
    qo, ko = _offsets(rq), _offsets(rk)
    T, Tk = qo[-1] + 9, ko[-1] + 5   # rows past the table's end keep their sentinels
    desc = _descriptor(T, Tk, D, mode, H, causal, lowMid=lowMid)
    x = _inputs(desc, G, T, Tk, seed)
    with window_block:
        if form == "packed":
            return run_packed(desc, G, x, qo, ko)
        from tests.test_paged_kv import PagedRun, build_pool
        Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, 16 if seed % 2 else 64, np.random.default_rng(seed))
        paged = PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, rk, table)
        paged.encode()
        return paged.results()


def dump(out_dir, timed, names, cases=CASES, run=run_case, functions=lambda case: instantiations(*case[:2], case[7]),
         backend="simtFP32"):
    """Runs `cases` through `run`, each of whose kernels must be on `backend`; functions(case): its entry functions"""
    import torch
    import mfa_b200 as mfa
    os.makedirs(out_dir, exist_ok=True)
    info = {"library": mfa.library_path(), "version": mfa.version(), "timed": timed, "cases": {}}
    for i, (name, case) in enumerate(cases.items()):
        if names and name not in names:
            continue
        record = {}
        with recorded(mfa, torch, record, timed):
            out = run(mfa, torch, 3000 + i, timed, *case)
        bad = {kind: r["backend"] for kind, r in record.items() if r["backend"] != backend}
        assert not bad and len(record) == (1 if case[0] == "paged" else 3), (name, record)
        if not timed:
            for key, array in out.items():
                np.save(os.path.join(out_dir, f"{name}_{key}.npy"), array)
        digests = {key: hashlib.sha256(array.tobytes()).hexdigest() for key, array in out.items()}
        info["cases"][name] = {"instantiations": functions(case), "kernels": record, "outputs": digests}
        print(name, json.dumps(record), flush=True)
    with open(os.path.join(out_dir, "shapes.json"), "w") as f:
        json.dump(info, f, indent=1)


def compare(a, b):
    ok = True
    infos = []
    for d in (a, b):
        with open(os.path.join(d, "shapes.json")) as f:
            infos.append(json.load(f))
    for name in infos[0]["cases"]:
        ca, cb = (info["cases"].get(name) for info in infos)
        if ca is None or cb is None:
            print(f"{name}: MISSING")
            ok = False
            continue
        for kind in sorted(set(ca["kernels"]) | set(cb["kernels"])):
            ka, kb = ca["kernels"].get(kind, {}), cb["kernels"].get(kind, {})
            same = all(ka.get(k) == kb.get(k) for k in ("backend", "launches"))
            line = f"{name} {kind}: launches {'identical' if same else f'DIFFERENT {ka} -> {kb}'}"
            if "ms" in ka and "ms" in kb:
                line += f", {ka['ms']:.3f} -> {kb['ms']:.3f} ms, new/old {kb['ms'] / ka['ms']:.3f}"
            print(line)
            ok &= same
        if sorted(ca["outputs"]) != sorted(cb["outputs"]):
            print(f"{name}: DIFFERENT outputs {sorted(ca['outputs'])} -> {sorted(cb['outputs'])}")
            ok = False
            continue
        if infos[0]["timed"] or infos[1]["timed"]:   # digests of the arrays only
            for out in ca["outputs"]:
                same = ca["outputs"][out] == cb["outputs"][out]
                print(f"{name} {out}: {'identical' if same else 'DIFFERENT'} (digest)")
                ok &= same
            continue
        for out in ca["outputs"]:
            x, y = (np.load(os.path.join(d, f"{name}_{out}.npy")) for d in (a, b))
            same = x.shape == y.shape and np.array_equal(x, y, equal_nan=True)
            diff = 0.0 if same or x.shape != y.shape else float(np.nanmax(np.abs(x.astype(np.float64) - y)))
            print(f"{name} {out}: {'identical' if same else f'DIFFERENT (max |diff| {diff:.3e})'}")
            ok &= same
    return ok


def main(**cases):
    """The command line; `cases`: dump's cases, run, functions and backend (default: the SIMT cases)"""
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory to write the arrays (with --time: the timings) to")
    ap.add_argument("--time", action="store_true", help="time each kernel type at a user's sizes; save digests only")
    ap.add_argument("--case", action="append", choices=list(cases.get("cases", CASES)),
                    help="run only this case (repeatable)")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"), help="compare the cases DIR_A holds")
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    if not args.out:
        ap.error("--out or --compare is required")
    dump(args.out, args.time, args.case, **cases)


if __name__ == "__main__":
    main()
