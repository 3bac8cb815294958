"""FP8 K/V (encode(..., paged=, split=, fp8=FP8KV())) against 16-bit pools: device time of one paged forward, BF16 Q,
H = 32 query heads, causal, shuffled pages ([num_pages][P][Hkv][D]), each under the library's split plan
(split=SplitKV()), which does not depend on the K/V element type.
  decode    S sequences of one query over Cs cached keys, G query heads per K/V head, D, P (the DESIGN section 8 rows)
  chunk     Rs = 16 queries per sequence
  window    the (4095, 0) windowed decode over 32768 keys
  prefill   a chunked-prefill row: 8 sequences of 1024 queries over 4096 keys
Calls alternate after a warm-up (CUDA events, eager launches), so that clock and thermal drift hit both alike; each is
repeated --reps times and reported as median, min and max.  Each row gives the K/V bytes one call must read (FP8: one
byte per element), that rate and its share of HBM3's 3.35 TB/s, and whether the FP8 output equals the 16-bit call's bit
for bit (the 16-bit pools hold the FP8 values, scales are NULL).  The card name and power limit are read in the same run.
--fp16 runs Q (and the 16-bit pools) in FP16 instead, whose conversion from E4M3 is one instruction per two values
(BF16 goes through FP32).
Usage (on an H100):  python scripts/bench_fp8_kv.py [--out-dir DIR] [--reps 5] [--quick] [--fp16]; the JSON goes to
DIR/bench_fp8_kv.json or bench_fp8_kv_fp16.json (default: a bench_fp8_kv directory under the system temporary directory)."""
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
from scripts.bench_gqa import card, events_timer  # noqa: E402

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
H = 32
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


class Case:
    """S sequences of Rs queries over Cs keys in shuffled pages of P keys, as FP8 bytes and as 16-bit pools holding
    the same values."""

    def __init__(self, S, Rs, Cs, G, D, page_size, window=None, dtype=torch.bfloat16):
        self.S, self.Rs, self.Cs, self.Hkv, self.D = S, Rs, Cs, H // G, D
        T = S * Rs
        desc = mfa.AttentionDescriptor()
        desc.lowPrecisionInputs = True
        desc.inputPrecisionOverride = P.BF16 if dtype == torch.bfloat16 else P.FP16
        desc.matrixDimensions = (T, S * Cs, D)
        desc.transposeState = (False,) * 4
        desc.batchCount = H
        desc.causal = True
        self.kernel = mfa.AttentionKernel.cached(desc, KT.forward, window=window)
        self.q = torch.randn(H, T, D, device="cuda").to(dtype)
        self.O, self.L = torch.empty(H, T, D, device="cuda"), torch.empty(H, T, device="cuda")
        self.rows = torch.arange(0, T + 1, Rs, dtype=torch.int32, device="cuda")
        per_seq = -(-Cs // page_size)
        num_pages = S * per_seq + 8
        self.k8, self.v8 = ((torch.randn(num_pages * page_size, self.Hkv, D, device="cuda") * 4)
                            .to(torch.float8_e4m3fn).view(torch.uint8) for _ in range(2))
        self.k16, self.v16 = (p.view(torch.float8_e4m3fn).to(dtype) for p in (self.k8, self.v8))
        self.page_table = torch.randperm(num_pages, device="cuda")[:S * per_seq].view(S, per_seq).to(torch.int32)
        self.lengths = torch.full((S,), Cs, dtype=torch.int32, device="cuda")
        self.paged = mfa.PagedKV(S, Rs, self.rows.data_ptr(), self.lengths.data_ptr(), self.page_table.data_ptr(),
                                 per_seq, page_size)
        self.c = mfa.FunctionConstantValues()
        self.c._c.row, self.c._c.column, self.c._c.batch_count, self.c._c.kv_group = T, num_pages * page_size, H, G
        torch.cuda.synchronize()   # (built on the default stream; the calls run on another)

    def call(self, fp8):
        k, v = (self.k8, self.v8) if fp8 else (self.k16, self.v16)
        ptrs = {Op.Q: self.q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: self.O.data_ptr(),
                Op.L: self.L.data_ptr()}
        extra = {"fp8": mfa.FP8KV()} if fp8 else {}
        return lambda s: self.kernel.encode(self.c, ptrs, s, paged=self.paged, split=mfa.SplitKV(), **extra)

    def kv_bytes(self, element_bytes, window=None):
        keys = self.Cs if window is None else min(self.Cs, window + self.Rs)
        return 2 * self.S * keys * self.Hkv * self.D * element_bytes


def measure(kind, S, Rs, Cs, G, D, page_size, reps, window=None, launches=3, dtype=torch.bfloat16):
    torch.manual_seed(0)
    case = Case(S, Rs, Cs, G, D, page_size, None if window is None else (window, 0), dtype)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    calls = {"16bit": case.call(False), "fp8": case.call(True)}
    plan = case.kernel.splitPlan(case.c, paged=case.paged, split=mfa.SplitKV())
    outputs = {}
    with torch.cuda.stream(stream):
        for name, fn in calls.items():
            case.O.fill_(float("nan"))
            case.L.fill_(float("nan"))
            fn(s)
            stream.synchronize()
            outputs[name] = (case.O.clone(), case.L.clone())
    timers = {name: events_timer(lambda fn=fn: fn(s), stream, launches) for name, fn in calls.items()}
    for fn in timers.values():   # warm-up
        fn()
    us = {name: [] for name in timers}
    for _ in range(reps):
        for name, fn in timers.items():
            us[name].append(fn())
    row = {"kind": kind, "S": S, "Rs": Rs, "Cs": Cs, "H": H, "G": G, "D": D, "page_size": page_size, "window": window,
           "causal": True, "q_dtype": "BF16" if dtype == torch.bfloat16 else "FP16", "reps": reps,
           "plan_splits": plan.splits, "plan_heads_per_tile": plan.heads_per_tile,
           "fp8_equals_16bit": all(torch.equal(a, b) for a, b in zip(outputs["fp8"], outputs["16bit"]))}
    for name, xs in us.items():
        med = statistics.median(xs)
        rate = case.kv_bytes(1 if name == "fp8" else 2, window) / (med * 1e-6)
        row[name] = {"us": round(med, 2), "us_min": round(min(xs), 2), "us_max": round(max(xs), 2),
                     "kv_tb_per_s": round(rate / 1e12, 3), "of_hbm_peak": round(rate / HBM_BYTES_PER_S, 3)}
    b = row["16bit"]
    row["fp8_over_16bit"] = round(row["fp8"]["us"] / b["us"], 3)
    row["16bit_spread"] = round((b["us_max"] - b["us_min"]) / b["us"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_fp8_kv"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--quick", action="store_true", help="a subset of the decode rows")
    ap.add_argument("--fp16", action="store_true", help="FP16 Q and 16-bit pools instead of BF16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fp8_kv.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "cases": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    rows = []
    for S, Cs in ((1, 4096), (1, 32768), (8, 4096), (8, 32768), (64, 4096)):
        for G in (1, 4, 8):
            for D in (64, 128):
                for page_size in (16, 256):
                    if args.quick and (G == 4 or page_size == 16):
                        continue
                    rows.append(("decode", S, 1, Cs, G, D, page_size, None))
    rows.append(("chunk", 8, 16, 4096, 8, 128, 256, None))
    rows.append(("window", 1, 1, 32768, 8, 128, 256, 4095))
    rows.append(("window", 8, 1, 32768, 8, 128, 256, 4095))
    rows.append(("prefill", 8, 1024, 4096, 8, 128, 256, None))
    for kind, S, Rs, Cs, G, D, page_size, window in rows:
        row = measure(kind, S, Rs, Cs, G, D, page_size, args.reps, window=window,
                      dtype=torch.float16 if args.fp16 else torch.bfloat16)
        print(json.dumps(row), flush=True)
        result["cases"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_fp8_kv_fp16.json" if args.fp16 else "bench_fp8_kv.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
