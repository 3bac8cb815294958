"""Packed variable-length sequences against the calls they replace: device time of the forward, dQ and dK/dV kernels
of one packed call (AttentionKernel.encode(..., sequences=)) over 32768 tokens, H = 32 query heads, D = 128, bf16,
causal and not, G = 1 and 8 query heads per K/V head.
  uniform  8 sequences of 4096, against the fixed-length batched call (batch H * 8, the same work)
  mixed    a seeded mix of lengths from 64 to 8192, against one encode per sequence (today's workaround)
The packed call and its comparison alternate after a warm-up (CUDA events, eager launches), so that clock and thermal
drift hit both alike; each is repeated --reps times and reported as median, min and max.  TFLOP/s count the visible
(query, key) pairs of every sequence and head.  The card name and power limit are read in the same run.
Usage (on an H100):  python scripts/bench_varlen.py [--out-dir DIR] [--reps 5]; the JSON goes to DIR/bench_varlen.json
(default: a bench_varlen directory under the system temporary directory)."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mfa_b200 as mfa  # noqa: E402
from scripts.bench_gqa import GEMM_FLOPS, card, events_timer, visible_pairs  # noqa: E402

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
TOKENS, H, D = 32768, 32, 128


def mixed_lengths(seed=0, lo=64, hi=8192):
    """Seeded lengths in [lo, hi] that sum to TOKENS (the last one takes the remainder)."""
    rng = np.random.default_rng(seed)
    lengths = []
    while sum(lengths) < TOKENS:
        n = int(rng.integers(lo, hi + 1))
        left = TOKENS - sum(lengths)
        lengths.append(n if left - n >= lo else left)
    return lengths


def descriptor(R, C, batch, causal):
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = P.BF16
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = (False,) * 4
    desc.batchCount = batch
    desc.causal = causal
    return desc


class Call:
    """One encode of every kernel type on its own buffers: `lengths` packed (sequences=), or a fixed R x C call."""

    def __init__(self, R, batch, G, causal, lengths=None):
        self.desc = descriptor(R, R, batch, causal)
        self.c = mfa.FunctionConstantValues()
        self.desc.setFunctionConstants(self.c)
        self.c.kvGroup = G
        self.kernels = {t: mfa.AttentionKernel.cached(self.desc, t) for t in KT}
        q, do = (torch.randn(batch, R, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        k, v = (torch.randn(batch // G, R, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        self.tensors = {Op.Q: q, Op.dO: do, Op.K: k, Op.V: v, Op.O: torch.empty(batch, R, D, device="cuda"),
                        Op.dQ: torch.empty(batch, R, D, device="cuda"), Op.L: torch.zeros(batch, R, device="cuda"),
                        Op.D: torch.zeros(batch, R, device="cuda"),
                        Op.dK: torch.empty(batch // G, R, D, device="cuda"),
                        Op.dV: torch.empty(batch // G, R, D, device="cuda")}
        self.ptrs = {op: t.data_ptr() for op, t in self.tensors.items()}
        self.table = None
        if lengths is not None:
            self.offsets = torch.tensor([0] + list(np.cumsum(lengths)), dtype=torch.int32, device="cuda")
            self.table = mfa.SequenceTable(len(lengths), max(lengths), max(lengths), self.offsets.data_ptr(),
                                           self.offsets.data_ptr())

    def encode(self, t, stream):
        self.kernels[t].encode(self.c, self.ptrs, stream, sequences=self.table)


def measure(kind, G, causal, reps, launches=3):
    torch.manual_seed(0)
    lengths = [4096] * 8 if kind == "uniform" else mixed_lengths()
    packed = Call(TOKENS, H, G, causal, lengths)
    if kind == "uniform":   # the same work as one fixed-length batched call
        others = [Call(4096, H * 8, G, causal)]
    else:                   # one call per sequence
        others = [Call(n, H, G, causal) for n in lengths]
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    pairs = sum(visible_pairs(n, n, causal) for n in lengths)
    row = {"kind": kind, "tokens": TOKENS, "sequences": len(lengths), "lengths": lengths, "H": H, "D": D, "G": G,
           "causal": causal, "dtype": "BF16", "reps": reps}
    with torch.cuda.stream(stream):
        for t in KT:   # forward first: dQ and dK/dV read its L
            packed.encode(t, s)
            for o in others:
                o.encode(t, s)
        stream.synchronize()
    comparison = "batched" if kind == "uniform" else "per_sequence_loop"
    for t in KT:
        def other_calls():
            for o in others:
                o.encode(t, s)
        timers = {"packed": events_timer(lambda: packed.encode(t, s), stream, launches),
                  comparison: events_timer(other_calls, stream, launches)}
        for fn in timers.values():   # warm-up
            fn()
        us = {name: [] for name in timers}
        for _ in range(reps):
            for name, fn in timers.items():
                us[name].append(fn())
        r = {}
        for name, xs in us.items():
            med = statistics.median(xs)
            r[name] = {"us": round(med, 1), "us_min": round(min(xs), 1), "us_max": round(max(xs), 1),
                       "tflops": round(GEMM_FLOPS[t] * pairs * D * H / med / 1e6, 1)}
        r["packed_over_" + comparison] = round(r["packed"]["us"] / r[comparison]["us"], 3)
        r["launches"] = {"packed": packed.kernels[t].launchCount(packed.c, packed.table),
                         comparison: sum(o.kernels[t].launchCount(o.c) for o in others)}
        row[t.name] = r
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_varlen"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_varlen.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "cases": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    for kind in ("uniform", "mixed"):
        for causal in (False, True):
            for G in (1, 8):
                row = measure(kind, G, causal, args.reps)
                print(json.dumps({k: v for k, v in row.items() if k != "lengths"}), flush=True)
                result["cases"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_varlen.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
