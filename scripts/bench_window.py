"""Sliding-window attention (AttentionKernel(kd, window=(left, right))) against the kernels it replaces: device time of
each kernel, bf16, D = 128, H = 32 query heads (G = 1 for prefill, G = 4 for decode).
  prefill   N = 8192 and 32768, causal window (4095, 0) against causal: forward, dQ and dK/dV
  band      (128, 128) at N = 8192 against unmasked: forward, dQ and dK/dV
  decode    S = 64 sequences of one query over Cs = 32768 cached keys in pages of P = 16, 64 and 256, window (4095, 0)
            against the full-context paged call; at D = 64 too, for P = 16 and 256
Calls alternate after a warm-up (CUDA events, eager launches), so that clock and thermal drift hit both alike; each is
repeated --reps times and reported as median, min and max.  Prefill and band rows give TFLOP/s over the visible
(query, key) pairs of each call; decode rows give the K/V bytes each call must read (the keys its window covers) per
second.  The card name and power limit are read in the same run.
Usage (on an H100):  python scripts/bench_window.py [--out-dir DIR] [--reps 5]; the JSON goes to DIR/bench_window.json
(default: a bench_window directory under the system temporary directory)."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mfa_b200 as mfa  # noqa: E402
from scripts.bench_gqa import GEMM_FLOPS, card, events_timer  # noqa: E402

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
H, D = 32, 128


def band_pairs(R, C, left, right):
    """(query, key) pairs a band sees (-1: unbounded side), counted per row in closed form"""
    delta, total = C - R, 0
    for i in range(R):
        lo = 0 if left < 0 else max(0, i + delta - left)
        hi = C - 1 if right < 0 else min(C - 1, i + delta + right)
        total += max(0, hi - lo + 1)
    return total


def _descriptor(R, C, causal, batch=H, D=D):
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = P.BF16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = (False,) * 4
    desc.batchCount = batch
    desc.causal = causal
    return desc


def _summary(samples):
    return {"median_us": statistics.median(samples), "min_us": min(samples), "max_us": max(samples)}


def prefill(N, causal, window, reps, launches=2):
    """The three kernels at N x N with and without the window; rows per kernel type."""
    desc = _descriptor(N, N, causal)
    c = mfa.FunctionConstantValues()
    desc.setFunctionConstants(c)
    bf = lambda *shape: torch.randn(*shape, device="cuda").to(torch.bfloat16)  # noqa: E731
    f32 = lambda *shape: torch.empty(*shape, device="cuda")  # noqa: E731
    inputs = {Op.Q: bf(H, N, D), Op.K: bf(H, N, D), Op.V: bf(H, N, D), Op.dO: bf(H, N, D)}
    # each variant has outputs of its own, so that its backward reads the L and D of its own mask
    ptrs, keep = {}, []
    for name in ("baseline", "windowed"):
        out = {Op.O: f32(H, N, D), Op.L: f32(H, N), Op.D: f32(H, N), Op.dQ: f32(H, N, D), Op.dK: f32(H, N, D),
               Op.dV: f32(H, N, D)}
        keep.append(out)
        ptrs[name] = {op: t.data_ptr() for op, t in {**inputs, **out}.items()}
    stream = torch.cuda.Stream()
    rows = []
    for t in KT:
        kernels = {"baseline": mfa.AttentionKernel.cached(desc, t),
                   "windowed": mfa.AttentionKernel.cached(desc, t, window=window)}
        timers = {name: events_timer(lambda k=k, n=name: k.encode(c, ptrs[n], stream.cuda_stream), stream, launches)
                  for name, k in kernels.items()}
        for timer in timers.values():   # warm-up (the backward reads the L and D its variant's forward left)
            timer()
        samples = {name: [] for name in timers}
        for _ in range(reps):
            for name, timer in timers.items():
                samples[name].append(timer())
        left, right = window
        pairs = {"baseline": band_pairs(N, N, -1, 0 if causal else -1), "windowed": band_pairs(N, N, left, right)}
        row = {"kind": "prefill" if causal else "band", "N": N, "type": t.name, "window": list(window)}
        for name in timers:
            s = _summary(samples[name])
            s["tflops"] = GEMM_FLOPS[t] * D * pairs[name] * H / (s["median_us"] * 1e-6) / 1e12
            row[name] = s
        row["ratio"] = row["windowed"]["median_us"] / row["baseline"]["median_us"]
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def decode(page_size, window, reps, S=64, Cs=32768, G=4, D=D, launches=10):
    """One decode step of S sequences over a paged cache, full context against the window."""
    Hkv = H // G
    pages_per_seq = Cs // page_size
    num_pages = S * pages_per_seq
    desc = _descriptor(S, num_pages * page_size, True, D=D)
    c = mfa.FunctionConstantValues()
    desc.setFunctionConstants(c)
    c.kvGroup = G
    q = torch.randn(H, S, D, device="cuda").to(torch.bfloat16)
    k_pool, v_pool = (torch.randn(num_pages, page_size, Hkv, D, device="cuda").to(torch.bfloat16) for _ in range(2))
    O, L = torch.empty(H, S, D, device="cuda"), torch.empty(H, S, device="cuda")
    rows_t = torch.arange(0, S + 1, dtype=torch.int32, device="cuda")
    lengths = torch.full((S,), Cs, dtype=torch.int32, device="cuda")
    table = torch.randperm(num_pages, device="cuda").to(torch.int32).reshape(S, pages_per_seq)
    paged = mfa.PagedKV(S, 1, rows_t.data_ptr(), lengths.data_ptr(), table.data_ptr(), pages_per_seq, page_size)
    ptrs = {Op.Q: q.data_ptr(), Op.K: k_pool.data_ptr(), Op.V: v_pool.data_ptr(), Op.O: O.data_ptr(), Op.L: L.data_ptr()}
    stream = torch.cuda.Stream()
    kernels = {"baseline": mfa.AttentionKernel.cached(desc, KT.forward),
               "windowed": mfa.AttentionKernel.cached(desc, KT.forward, window=window)}
    timers = {name: events_timer(lambda k=k: k.encode(c, ptrs, stream.cuda_stream, paged=paged), stream, launches)
              for name, k in kernels.items()}
    for timer in timers.values():
        timer()
    samples = {name: [] for name in timers}
    for _ in range(reps):
        for name, timer in timers.items():
            samples[name].append(timer())
    keys = {"baseline": Cs, "windowed": min(Cs, window[0] + 1)}
    row = {"kind": "decode", "S": S, "Cs": Cs, "G": G, "D": D, "page_size": page_size, "window": list(window)}
    for name in timers:
        s = _summary(samples[name])
        s["kv_bytes"] = 2 * S * keys[name] * Hkv * D * 2
        s["bytes_per_s"] = s["kv_bytes"] / (s["median_us"] * 1e-6)
        row[name] = s
    row["ratio"] = row["windowed"]["median_us"] / row["baseline"]["median_us"]
    print(json.dumps(row), flush=True)
    return [row]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_window"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_window.py measures on the GPU"
    torch.manual_seed(0)
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for N in (8192, 32768):
        rows += prefill(N, True, (4095, 0), args.reps)
    rows += prefill(8192, False, (128, 128), args.reps)
    for page_size in (16, 64, 256):
        rows += decode(page_size, (4095, 0), args.reps)
    # D = 64: the windowed paged forward takes 138 registers there (one CTA per SM), the full-context one 126
    for page_size in (16, 256):
        rows += decode(page_size, (4095, 0), args.reps, D=64)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "bench_window.json"), "w") as f:
        json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
