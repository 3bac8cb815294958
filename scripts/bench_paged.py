"""The forward over a paged K/V cache (AttentionKernel.encode(..., paged=)) against the calls it replaces: device time
of one forward, bf16, D = 128, H = 32 query heads, G = 1 and 8 query heads per K/V head, page sizes 16, 64 and 256,
causal and not.  The pools are [num_pages][P][Hkv][D] with shuffled pages.
  prefill  8 sequences of 4096 queries over their 4096 keys: paged against the packed call (sequences=) on the same keys
           stored contiguously, head-major
  decode   S = 64 and S = 8 sequences of Rs = 1 (and Rs = 16) queries over Cs = 4096 cached keys: paged against
           (a) the packed call on contiguous keys and (b) gather + packed: copying every sequence's pages into a fresh
           contiguous head-major K and V, then the packed call (what a caller does without paging support)
Calls alternate after a warm-up (CUDA events, eager launches), so that clock and thermal drift hit all alike; each is
repeated --reps times and reported as median, min and max.  Prefill rows give TFLOP/s of the visible (query, key)
pairs; decode rows give the K/V bytes each call must read per second, and that rate over HBM3's 3.35 TB/s.  The card
name and power limit are read in the same run.
Usage (on an H100):  python scripts/bench_paged.py [--out-dir DIR] [--reps 5]; the JSON goes to DIR/bench_paged.json
(default: a bench_paged directory under the system temporary directory)."""
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
from scripts.bench_gqa import GEMM_FLOPS, card, events_timer, visible_pairs  # noqa: E402

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision
H, D = 32, 128
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


class Case:
    """S sequences of Rs queries over Cs keys each, K/V both contiguous ([Hkv][S * Cs][D]) and paged (shuffled pages
    of a pool [num_pages][P][Hkv][D] holding the same keys), and the buffers of the three calls."""

    def __init__(self, S, Rs, Cs, G, page_size, causal):
        self.S, self.Rs, self.Cs, self.Hkv = S, Rs, Cs, H // G
        T, Tk = S * Rs, S * Cs
        desc = mfa.AttentionDescriptor()
        desc.lowPrecisionInputs = True
        desc.inputPrecisionOverride = P.BF16
        desc.matrixDimensions = (T, Tk, D)
        desc.transposeState = (False,) * 4
        desc.batchCount = H
        desc.causal = causal
        self.kernel = mfa.AttentionKernel.cached(desc, KT.forward)
        self.c = mfa.FunctionConstantValues()
        desc.setFunctionConstants(self.c)
        self.c.kvGroup = G
        q = torch.randn(H, T, D, device="cuda").to(torch.bfloat16)
        self.k, self.v = (torch.randn(self.Hkv, Tk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        self.O, self.L = torch.empty(H, T, D, device="cuda"), torch.empty(H, T, device="cuda")
        self.rows = torch.arange(0, T + 1, Rs, dtype=torch.int32, device="cuda")
        self.columns = torch.arange(0, Tk + 1, Cs, dtype=torch.int32, device="cuda")
        self.packed_table = mfa.SequenceTable(S, Rs, Cs, self.rows.data_ptr(), self.columns.data_ptr())
        self.packed_ptrs = {Op.Q: q.data_ptr(), Op.K: self.k.data_ptr(), Op.V: self.v.data_ptr(),
                            Op.O: self.O.data_ptr(), Op.L: self.L.data_ptr()}
        # the pools: every sequence's ceil(Cs / P) pages, shuffled, plus a few spare ones
        per_seq = -(-Cs // page_size)
        num_pages = S * per_seq + 8
        self.page_table = torch.randperm(num_pages, device="cuda")[:S * per_seq].view(S, per_seq).to(torch.int32)
        key = torch.arange(Cs, device="cuda")
        self.slots = (self.page_table.long()[:, key // page_size] * page_size + key % page_size).reshape(-1)
        self.k_pool, self.v_pool = (torch.zeros(num_pages * page_size, self.Hkv, D, device="cuda",
                                                dtype=torch.bfloat16) for _ in range(2))
        self.k_pool[self.slots] = self.k.transpose(0, 1)
        self.v_pool[self.slots] = self.v.transpose(0, 1)
        self.lengths = torch.full((S,), Cs, dtype=torch.int32, device="cuda")
        self.paged = mfa.PagedKV(S, Rs, self.rows.data_ptr(), self.lengths.data_ptr(), self.page_table.data_ptr(),
                                 per_seq, page_size)
        self.paged_c = mfa.FunctionConstantValues()
        self.paged_c._c.row, self.paged_c._c.column = T, num_pages * page_size
        self.paged_c._c.batch_count, self.paged_c._c.kv_group = H, G
        self.paged_ptrs = {**self.packed_ptrs, Op.K: self.k_pool.data_ptr(), Op.V: self.v_pool.data_ptr()}
        self.gathered_k, self.gathered_v = (torch.empty(Tk, self.Hkv, D, device="cuda", dtype=torch.bfloat16)
                                            for _ in range(2))
        torch.cuda.synchronize()   # (built on the default stream; the calls run on another)

    def run_paged(self, s):
        self.kernel.encode(self.paged_c, self.paged_ptrs, s, paged=self.paged)

    def run_packed(self, s):
        self.kernel.encode(self.c, self.packed_ptrs, s, sequences=self.packed_table)

    def run_gather_packed(self, s):
        # (writes into the contiguous buffers the packed call reads: a fresh copy of every sequence's keys and values)
        torch.index_select(self.k_pool, 0, self.slots, out=self.gathered_k)
        torch.index_select(self.v_pool, 0, self.slots, out=self.gathered_v)
        self.k.copy_(self.gathered_k.transpose(0, 1))
        self.v.copy_(self.gathered_v.transpose(0, 1))
        self.run_packed(s)

    def kv_bytes(self):
        return 2 * self.S * self.Cs * self.Hkv * D * 2


def measure(kind, S, Rs, Cs, G, page_size, causal, reps, launches=3):
    torch.manual_seed(0)
    case = Case(S, Rs, Cs, G, page_size, causal)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    calls = {"paged": case.run_paged, "packed": case.run_packed}
    if kind == "decode":
        calls["gather_packed"] = case.run_gather_packed
    with torch.cuda.stream(stream):
        outputs = {}
        for name, fn in calls.items():
            case.O.fill_(float("nan"))
            fn(s)
            stream.synchronize()
            outputs[name] = case.O.clone()
        stream.synchronize()
    # the calls compute the same thing: paged and packed bit for bit
    same = all(torch.equal(outputs["paged"], o) for o in outputs.values())
    timers = {name: events_timer(lambda fn=fn: fn(s), stream, launches) for name, fn in calls.items()}
    for fn in timers.values():   # warm-up
        fn()
    us = {name: [] for name in timers}
    for _ in range(reps):
        for name, fn in timers.items():
            us[name].append(fn())
    row = {"kind": kind, "S": S, "Rs": Rs, "Cs": Cs, "H": H, "D": D, "G": G, "page_size": page_size, "causal": causal,
           "dtype": "BF16", "reps": reps, "paged_equals_packed": same}
    pairs = S * visible_pairs(Rs, Cs, causal)
    for name, xs in us.items():
        med = statistics.median(xs)
        r = {"us": round(med, 2), "us_min": round(min(xs), 2), "us_max": round(max(xs), 2)}
        if kind == "prefill":
            r["tflops"] = round(GEMM_FLOPS[KT.forward] * pairs * D * H / med / 1e6, 1)
        else:
            rate = case.kv_bytes() / (med * 1e-6)
            r["kv_tb_per_s"] = round(rate / 1e12, 3)
            r["of_hbm_peak"] = round(rate / HBM_BYTES_PER_S, 3)
        row[name] = r
    for name in us:
        if name != "paged":
            row["paged_over_" + name] = round(row["paged"]["us"] / row[name]["us"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_paged"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_paged.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "cases": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    shapes = [("prefill", 8, 4096, 4096), ("decode", 64, 1, 4096), ("decode", 8, 1, 4096), ("decode", 64, 16, 4096),
              ("decode", 8, 16, 4096)]
    for kind, S, Rs, Cs in shapes:
        for causal in (False, True):
            for G in (1, 8):
                for page_size in (16, 64, 256):
                    row = measure(kind, S, Rs, Cs, G, page_size, causal, args.reps)
                    print(json.dumps(row), flush=True)
                    result["cases"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_paged.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
