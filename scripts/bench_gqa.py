"""Grouped-query attention against the workaround it replaces: device time of the forward, dQ and dK/dV kernels with
K/V shared by G query heads (FunctionConstantValues.kvGroup = G), and of the same library on K/V expanded with
torch.repeat_interleave, whose per-head dK / dV are then summed per group with torch.  The expansion and the sum are
timed on their own and reported beside the kernel time.  Grouped and expanded calls alternate after a warm-up (CUDA
events, eager launches), so that clock and thermal drift hit both alike.  TFLOP/s count the (query, key) pairs the mask
leaves visible, for all Hq query heads.  The card name and power limit are read (read-only nvidia-smi query) in the
same run; without a GPU the script fails.
Usage (on an H100):  python scripts/bench_gqa.py [--out-dir DIR] [--reps 5]; the JSON goes to DIR/bench_gqa.json
(default: a bench_gqa directory under the system temporary directory)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mfa_b200 as mfa  # noqa: E402

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
GEMM_FLOPS = {KT.forward: 4, KT.backwardQuery: 6, KT.backwardKeyValue: 8}  # per visible (query, key) pair and head column

# (R, C, D, Hq, G, causal, kernel types)
ALL = tuple(KT)
SHAPES = [(4096, 4096, 128, 64, G, causal, ALL) for causal in (False, True) for G in (1, 8, 64)] + [
    (8192, 8192, 128, 32, 4, False, ALL),
    (512, 16384, 128, 64, 8, True, (KT.forward,)),   # chunked prefill: 512 new queries against a 16384-key cache
]


def card():
    try:
        name, limit = subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
            text=True).strip().split(", ")
        return {"gpu": name, "power_limit": limit}
    except (OSError, subprocess.CalledProcessError, ValueError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def visible_pairs(R, C, causal):
    if not causal:
        return R * C
    return sum(max(0, min(C, i + C - R + 1)) for i in range(R))


def events_timer(fn, stream, launches):
    """us per call of fn() (which enqueues on `stream`), timed over `launches` calls with CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run():
        with torch.cuda.stream(stream):
            a.record(stream)
            for _ in range(launches):
                fn()
            b.record(stream)
            stream.synchronize()
        return a.elapsed_time(b) * 1e3 / launches
    return run


def measure(R, C, D, Hq, G, causal, types, reps, launches=3):
    torch.manual_seed(0)
    Hkv = Hq // G
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = P.BF16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = (False,) * 4
    desc.batchCount = Hq
    desc.causal = causal
    grouped_c, expanded_c = mfa.FunctionConstantValues(), mfa.FunctionConstantValues()
    desc.setFunctionConstants(grouped_c)
    desc.setFunctionConstants(expanded_c)
    grouped_c.kvGroup = G
    kernels = {t: mfa.AttentionKernel(desc.kernelDescriptor(t)) for t in types}

    q, do = (torch.randn(Hq, R, D, device="cuda").to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(Hkv, C, D, device="cuda").to(torch.bfloat16) for _ in range(2))
    k_exp, v_exp = k.repeat_interleave(G, dim=0), v.repeat_interleave(G, dim=0)
    common = {Op.Q: q, Op.dO: do, Op.O: torch.empty(Hq, R, D, device="cuda"), Op.dQ: torch.empty(Hq, R, D, device="cuda"),
              Op.L: torch.zeros(Hq, R, device="cuda"), Op.D: torch.zeros(Hq, R, device="cuda")}
    dk, dv = (torch.empty(Hkv, C, D, device="cuda") for _ in range(2))
    dk_exp, dv_exp = (torch.empty(Hq, C, D, device="cuda") for _ in range(2))
    grouped = {op: t.data_ptr() for op, t in {**common, Op.K: k, Op.V: v, Op.dK: dk, Op.dV: dv}.items()}
    expanded = {op: t.data_ptr() for op, t in {**common, Op.K: k_exp, Op.V: v_exp, Op.dK: dk_exp, Op.dV: dv_exp}.items()}
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def expand():
        k.repeat_interleave(G, dim=0)
        v.repeat_interleave(G, dim=0)

    def group_sum():
        dk_exp.view(Hkv, G, C, D).sum(dim=1)
        dv_exp.view(Hkv, G, C, D).sum(dim=1)

    row = {"R": R, "C": C, "D": D, "Hq": Hq, "Hkv": Hkv, "G": G, "causal": causal, "dtype": "BF16", "reps": reps}
    with torch.cuda.stream(stream):
        for t in types:   # forward first: dQ and dK/dV read its L
            kernels[t].encode(grouped_c, grouped, s)
            kernels[t].encode(expanded_c, expanded, s)
        stream.synchronize()
    flops_unit = visible_pairs(R, C, causal) * D * Hq
    for t in types:
        timers = {
            "gqa": events_timer(lambda: kernels[t].encode(grouped_c, grouped, s), stream, launches),
            "expanded_kernel": events_timer(lambda: kernels[t].encode(expanded_c, expanded, s), stream, launches),
            "expand": events_timer(expand, stream, launches),
        }
        if t == KT.backwardKeyValue:
            timers["group_sum"] = events_timer(group_sum, stream, launches)
        for fn in timers.values():   # warm-up
            fn()
        us = {name: [] for name in timers}
        for _ in range(reps):
            for name, fn in timers.items():
                us[name].append(fn())
        r = {}
        for name, xs in us.items():
            med = statistics.median(xs)
            r[name] = {"us": round(med, 1), "us_min": round(min(xs), 1), "us_max": round(max(xs), 1)}
            if name in ("gqa", "expanded_kernel"):
                r[name]["tflops"] = round(GEMM_FLOPS[t] * flops_unit / med / 1e6, 1)
        r["expanded_total_us"] = round(r["expanded_kernel"]["us"] + r["expand"]["us"] +
                                       (r["group_sum"]["us"] if "group_sum" in r else 0.0), 1)
        r["kernel_ratio"] = round(r["gqa"]["us"] / r["expanded_kernel"]["us"], 3)
        r["launches"] = {"gqa": kernels[t].launchCount(grouped_c), "expanded": kernels[t].launchCount(expanded_c)}
        row[t.name] = r
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_gqa"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gqa.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "shapes": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    for shape in SHAPES:
        row = measure(*shape, reps=args.reps)
        print(json.dumps(row), flush=True)
        result["shapes"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_gqa.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
