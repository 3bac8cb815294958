"""Split-KV decode (encode(..., split=SplitKV())) against the unsplit call it extends: device time of one forward,
bf16, H = 32 query heads, causal, on a paged cache with shuffled pages ([num_pages][P][Hkv][D]) and on packed
contiguous keys.
  decode    S sequences of Rs queries over Cs cached keys, G query heads per K/V head, D, P: the library's plan
            (num_splits = 0) and forced num_splits of 1, 2, 4, 8 and 16 against the existing encode(..., paged=)
  select    Rs = 127 and 128 at G = 8: either side of the rule that packs a group's query heads into one tile
  window    the (4095, 0) windowed paged decode over 32768 keys
  prefill   a packed chunked-prefill row (8 sequences of 1024 queries over 4096 keys), where the plan splits nothing
Calls alternate after a warm-up (CUDA events, eager launches), so that clock and thermal drift hit all alike; each is
repeated --reps times and reported as median, min and max.  Each row also gives the distinct K/V bytes one call must
read, that rate and its share of HBM3's 3.35 TB/s, and whether the library plan's output equals the existing call's
bit for bit when it plans one split.  The card name and power limit are read in the same run.
Usage (on an H100):  python scripts/bench_decode.py [--out-dir DIR] [--reps 5] [--quick]; the JSON goes to
DIR/bench_decode.json (default: a bench_decode directory under the system temporary directory)."""
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
FORCED = (1, 2, 4, 8, 16)


class Case:
    """S sequences of Rs queries over Cs keys; paged (shuffled pages of P keys) or packed (contiguous) K/V."""

    def __init__(self, S, Rs, Cs, G, D, page_size, paged, window=None):
        self.S, self.Rs, self.Cs, self.Hkv, self.D = S, Rs, Cs, H // G, D
        T, Tk = S * Rs, S * Cs
        desc = mfa.AttentionDescriptor()
        desc.lowPrecisionInputs = True
        desc.inputPrecisionOverride = P.BF16
        desc.matrixDimensions = (T, Tk, D)
        desc.transposeState = (False,) * 4
        desc.batchCount = H
        desc.causal = True
        self.kernel = mfa.AttentionKernel.cached(desc, KT.forward, window=window)
        q = torch.randn(H, T, D, device="cuda").to(torch.bfloat16)
        self.O, self.L = torch.empty(H, T, D, device="cuda"), torch.empty(H, T, device="cuda")
        self.rows = torch.arange(0, T + 1, Rs, dtype=torch.int32, device="cuda")
        self.c = mfa.FunctionConstantValues()
        self.c._c.row, self.c._c.batch_count, self.c._c.kv_group = T, H, G
        self.table = {}
        if paged:
            per_seq = -(-Cs // page_size)
            num_pages = S * per_seq + 8
            self.k, self.v = (torch.randn(num_pages * page_size, self.Hkv, D, device="cuda").to(torch.bfloat16)
                              for _ in range(2))
            self.page_table = torch.randperm(num_pages, device="cuda")[:S * per_seq].view(S, per_seq).to(torch.int32)
            self.lengths = torch.full((S,), Cs, dtype=torch.int32, device="cuda")
            self.table["paged"] = mfa.PagedKV(S, Rs, self.rows.data_ptr(), self.lengths.data_ptr(),
                                              self.page_table.data_ptr(), per_seq, page_size)
            self.c._c.column = num_pages * page_size
        else:
            self.k, self.v = (torch.randn(self.Hkv, Tk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
            self.columns = torch.arange(0, Tk + 1, Cs, dtype=torch.int32, device="cuda")
            self.table["sequences"] = mfa.SequenceTable(S, Rs, Cs, self.rows.data_ptr(), self.columns.data_ptr())
            self.c._c.column = Tk
        self.ptrs = {Op.Q: q.data_ptr(), Op.K: self.k.data_ptr(), Op.V: self.v.data_ptr(), Op.O: self.O.data_ptr(),
                     Op.L: self.L.data_ptr()}
        self.q = q
        torch.cuda.synchronize()   # (built on the default stream; the calls run on another)

    def call(self, split):
        return lambda s: self.kernel.encode(self.c, self.ptrs, s, split=split, **self.table)

    def plan(self, split):
        return self.kernel.splitPlan(self.c, split=split, **self.table)

    def kv_bytes(self, window=None):
        keys = self.Cs if window is None else min(self.Cs, window + self.Rs)
        return 2 * self.S * keys * self.Hkv * self.D * 2


def measure(kind, S, Rs, Cs, G, D, page_size, paged, reps, window=None, forced=FORCED, launches=3):
    torch.manual_seed(0)
    case = Case(S, Rs, Cs, G, D, page_size, paged, None if window is None else (window, 0))
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    calls = {"existing": case.call(None), "plan": case.call(mfa.SplitKV())}
    for n in forced:
        calls[f"split{n}"] = case.call(mfa.SplitKV(n))
    plan = case.plan(mfa.SplitKV())
    outputs = {}
    with torch.cuda.stream(stream):
        for name in ("existing", "plan"):
            case.O.fill_(float("nan"))
            calls[name](s)
            stream.synchronize()
            outputs[name] = case.O.clone()
    timers = {name: events_timer(lambda fn=fn: fn(s), stream, launches) for name, fn in calls.items()}
    for fn in timers.values():   # warm-up
        fn()
    us = {name: [] for name in timers}
    for _ in range(reps):
        for name, fn in timers.items():
            us[name].append(fn())
    row = {"kind": kind, "layout": "paged" if paged else "packed", "S": S, "Rs": Rs, "Cs": Cs, "H": H, "G": G, "D": D,
           "page_size": page_size if paged else None, "window": window, "causal": True, "dtype": "BF16", "reps": reps,
           "plan_splits": plan.splits, "plan_heads_per_tile": plan.heads_per_tile, "plan_grid": plan.grid_size,
           "plan_equals_existing": bool(torch.equal(outputs["plan"], outputs["existing"])),
           "max_abs_diff": float((outputs["plan"] - outputs["existing"]).abs().max())}
    kv = case.kv_bytes(window)
    for name, xs in us.items():
        med = statistics.median(xs)
        rate = kv / (med * 1e-6)
        row[name] = {"us": round(med, 2), "us_min": round(min(xs), 2), "us_max": round(max(xs), 2),
                     "kv_tb_per_s": round(rate / 1e12, 3), "of_hbm_peak": round(rate / HBM_BYTES_PER_S, 3)}
    ex = row["existing"]
    row["plan_over_existing"] = round(row["plan"]["us"] / ex["us"], 3)
    row["existing_spread"] = round((ex["us_max"] - ex["us_min"]) / ex["us"], 3)
    row["best_forced"] = min((n for n in forced), key=lambda n: row[f"split{n}"]["us"]) if forced else None
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_decode"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--quick", action="store_true", help="a subset of the decode rows")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_decode.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "cases": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    rows = []
    for S, Cs in ((1, 4096), (1, 32768), (8, 4096), (8, 32768), (64, 4096)):
        for Rs in (1, 16):
            for G in (1, 4, 8):
                for D in (64, 128):
                    for page_size in (16, 256):
                        if args.quick and (G == 4 or page_size == 16 or (D == 64 and Rs == 16)):
                            continue
                        rows.append(("decode", S, Rs, Cs, G, D, page_size, True, None))
    # both sides of the packing rule (query heads of a K/V head share a tile while max_row < 128)
    rows.append(("select", 8, 127, 4096, 8, 128, 256, True, None))
    rows.append(("select", 8, 128, 4096, 8, 128, 256, True, None))
    rows.append(("window", 1, 1, 32768, 8, 128, 256, True, 4095))
    rows.append(("window", 8, 1, 32768, 8, 128, 256, True, 4095))
    rows.append(("prefill", 8, 1024, 4096, 8, 128, 0, False, None))
    for kind, S, Rs, Cs, G, D, page_size, paged, window in rows:
        row = measure(kind, S, Rs, Cs, G, D, page_size, paged, args.reps, window=window)
        print(json.dumps(row), flush=True)
        result["cases"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_decode.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
