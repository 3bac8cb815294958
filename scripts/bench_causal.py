"""Causal against unmasked attention: device time of the forward, dQ and dK/dV kernels with and without the causal
mask, measured alternately (causal, unmasked, causal, ...) with CUDA events after a warm-up.  Shapes: the bench.py
headline (bf16, N = 4096, D = 128, 64 heads, eager launches) and one head of N = 4096 (CUDA graph of the launches, as
scripts/bench_single.py times it).  TFLOP/s count only the (query, key) pairs the mask leaves visible: N (N + 1) / 2 of
N^2 when causal.  The card name and power limit are read (read-only nvidia-smi query) in the same run.
Usage (on an H100):  python scripts/bench_causal.py [--out-dir DIR] [--reps 5]; the JSON goes to
DIR/bench_causal.json (default: a bench_causal directory under the system temporary directory)."""
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


def card():
    try:
        name, limit = subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
            text=True).strip().split(", ")
        return {"gpu": name, "power_limit": limit}
    except (OSError, subprocess.CalledProcessError, ValueError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def setup(N, D, H, causal):
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = P.BF16
    desc.matrixDimensions = (N, N, D)
    desc.transposeState = (False,) * 4
    desc.batchCount = H
    desc.causal = causal
    c = mfa.FunctionConstantValues()
    desc.setFunctionConstants(c)
    return {t: mfa.AttentionKernel(desc.kernelDescriptor(t)) for t in KT}, c


def buffers(N, D, H):
    torch.manual_seed(0)
    bufs = {op: torch.randn(H, N, D, device="cuda").to(torch.bfloat16) for op in (Op.Q, Op.K, Op.V, Op.dO)}
    for op in (Op.O, Op.dQ, Op.dK, Op.dV):
        bufs[op] = torch.empty(H, N, D, device="cuda")
    for op in (Op.L, Op.D):
        bufs[op] = torch.zeros(H, N, device="cuda")  # finite statistics, as a forward pass would leave them
    return bufs


def timer(kernel, c, ptrs, stream, graph, launches):
    """Returns a function that times `launches` encodes (eager, or replaying one captured graph of them) in us each."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g = None
    with torch.cuda.stream(stream):
        for _ in range(3):
            kernel.encode(c, ptrs, stream.cuda_stream)
        stream.synchronize()
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                for _ in range(launches):
                    kernel.encode(c, ptrs, stream.cuda_stream)
            g.replay()
            stream.synchronize()

    def run():
        with torch.cuda.stream(stream):
            a.record(stream)
            if g is not None:
                g.replay()
            else:
                for _ in range(launches):
                    kernel.encode(c, ptrs, stream.cuda_stream)
            b.record(stream)
            stream.synchronize()
        return a.elapsed_time(b) * 1e3 / launches
    return run


def measure(N, D, H, graph, launches, reps):
    bufs = buffers(N, D, H)
    ptrs = {op: t.data_ptr() for op, t in bufs.items()}
    stream = torch.cuda.Stream()
    out = {"N": N, "D": D, "heads": H, "dtype": "BF16", "timing": "cuda graph" if graph else "eager", "reps": reps}
    for t in KT:
        runs = {}
        for causal in (True, False):
            kernels, c = setup(N, D, H, causal)
            runs[causal] = (timer(kernels[t], c, ptrs, stream, graph, launches), kernels[t].launchCount(c))
        us = {True: [], False: []}
        for _ in range(reps):      # alternate, so that clock and thermal drift hit both alike
            for causal in (True, False):
                us[causal].append(runs[causal][0]())
        row = {}
        for causal in (True, False):
            pairs = N * (N + 1) // 2 if causal else N * N
            med = statistics.median(us[causal])
            row["causal" if causal else "unmasked"] = {
                "us": round(med, 2), "us_min": round(min(us[causal]), 2), "us_max": round(max(us[causal]), 2),
                "launches": runs[causal][1], "tflops": round(GEMM_FLOPS[t] * pairs * D * H / med / 1e6, 1)}
        row["ratio"] = round(row["causal"]["us"] / row["unmasked"]["us"], 3)
        out[t.name] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_causal"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "shapes": []}
    for N, D, H, graph, launches in ((4096, 128, 64, False, 5), (4096, 128, 1, True, 20)):
        row = measure(N, D, H, graph, launches, args.reps)
        print(json.dumps(row), flush=True)
        result["shapes"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_causal.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), "->", path)


if __name__ == "__main__":
    main()
