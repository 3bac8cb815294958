"""Paged K/V append (mfa.appendPagedKV) against the torch recipe it replaces: device time of writing one step's new keys
and values into shuffled page pools [num_pages][P][Hkv][D], Hkv = 8 K/V heads, D = 128, BF16 sources.
  decode    S sequences of Rs = 1 new token over Cs = 4096 cached keys, P = 16 and 256
  chunk     a chunked-prefill step: 8 sequences of 2048 new tokens (Cs = 4096)
each into BF16 pools (a copy) and into FP8 E4M3 pools with per-head scales (a quantization).  The torch recipe computes
the slot mapping on the device from the same tables (page_table[s][p // P] * P + p % P for p = Cs - Rs + i), so it
times kernels, not a Python loop; it then runs one index_copy_ per pool, after a saturating divide and conversion for
FP8.  Each row also times a whole decode step: the append followed by the split paged forward (32 query heads, causal,
the library's plan), against the torch recipe followed by the same forward.
Calls alternate after a warm-up (CUDA events, eager launches, --launches calls per timing), so that clock and thermal
drift hit both alike; each is repeated --reps times and reported as median, min and max.  Each row gives the bytes the
append must read and write, that rate and its share of HBM3's 3.35 TB/s, and whether the append's pool rows equal the
recipe's byte for byte.  The card name and power limit are read in the same run.
Usage (on an H100):  python scripts/bench_paged_append.py [--out-dir DIR] [--reps 5]; the JSON goes to
DIR/bench_paged_append.json (default: a bench_paged_append directory under the system temporary directory)."""
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
H, HKV, D = 32, 8, 128
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
E4M3_MAX = 448.0


class Case:
    def __init__(self, S, Rs, Cs, page_size, fp8):
        self.S, self.Rs, self.Cs, self.P, self.fp8 = S, Rs, Cs, page_size, fp8
        T = self.T = S * Rs
        per_seq = -(-Cs // page_size)
        num_pages = S * per_seq + 8
        self.pool_rows = num_pages * page_size
        pool_dtype = torch.uint8 if fp8 else torch.bfloat16
        self.k_pool, self.v_pool = (torch.zeros(self.pool_rows, HKV, D, dtype=pool_dtype, device="cuda")
                                    for _ in range(2))
        self.k_new, self.v_new = (torch.randn(T, HKV, D, device="cuda").to(torch.bfloat16) * 3 for _ in range(2))
        self.rows = torch.arange(0, T + 1, Rs, dtype=torch.int32, device="cuda")
        self.lengths = torch.full((S,), Cs, dtype=torch.int32, device="cuda")
        self.page_table = torch.randperm(num_pages, device="cuda")[:S * per_seq].view(S, per_seq).to(torch.int32)
        self.paged = mfa.PagedKV(S, Rs, self.rows.data_ptr(), self.lengths.data_ptr(), self.page_table.data_ptr(),
                                 per_seq, page_size)
        self.append_arg = mfa.PagedKVAppend(self.k_new.data_ptr(), self.v_new.data_ptr(), T, 0, HKV, D, self.pool_rows,
                                            P.BF16)
        self.scales = [torch.rand(HKV, device="cuda") * 0.05 + 0.01 for _ in range(2)]
        self.fp8_arg = mfa.FP8KV(self.scales[0].data_ptr(), self.scales[1].data_ptr()) if fp8 else None
        # the recipe's per-token constants: the token's sequence and its index among the sequence's new tokens
        self.token_seq = torch.arange(S, device="cuda").repeat_interleave(Rs)
        self.token_index = torch.arange(Rs, device="cuda").repeat(S)
        # the split paged forward of the step
        desc = mfa.AttentionDescriptor()
        desc.lowPrecisionInputs = True
        desc.inputPrecisionOverride = P.BF16
        desc.matrixDimensions = (T, self.pool_rows, D)
        desc.transposeState = (False,) * 4
        desc.batchCount = H
        desc.causal = True
        self.kernel = mfa.AttentionKernel.cached(desc, KT.forward)
        self.q = torch.randn(H, T, D, device="cuda").to(torch.bfloat16)
        self.O, self.L = torch.empty(H, T, D, device="cuda"), torch.empty(H, T, device="cuda")
        self.c = mfa.FunctionConstantValues()
        self.c._c.row, self.c._c.column, self.c._c.batch_count, self.c._c.kv_group = T, self.pool_rows, H, H // HKV
        torch.cuda.synchronize()   # (built on the default stream; the calls run on another)

    def slots(self):
        keys = (self.lengths[self.token_seq] - self.Rs + self.token_index).long()
        return self.page_table[self.token_seq, keys // self.P].long() * self.P + keys % self.P

    def append(self, s):
        mfa.appendPagedKV(self.paged, self.append_arg, self.k_pool.data_ptr(), self.v_pool.data_ptr(),
                          fp8=self.fp8_arg, stream=s)

    def recipe(self, s):
        slot = self.slots()
        for new, pool, scale in ((self.k_new, self.k_pool, self.scales[0]), (self.v_new, self.v_pool, self.scales[1])):
            if self.fp8:
                new = ((new.float() / scale[None, :, None]).clamp(-E4M3_MAX, E4M3_MAX)
                       .to(torch.float8_e4m3fn).view(torch.uint8))
            pool.index_copy_(0, slot, new)

    def forward(self, s):
        ptrs = {Op.Q: self.q.data_ptr(), Op.K: self.k_pool.data_ptr(), Op.V: self.v_pool.data_ptr(),
                Op.O: self.O.data_ptr(), Op.L: self.L.data_ptr()}
        extra = {"fp8": self.fp8_arg} if self.fp8 else {}
        self.kernel.encode(self.c, ptrs, s, paged=self.paged, split=mfa.SplitKV(), **extra)

    def bytes_moved(self):
        elements = self.T * HKV * D
        return 2 * elements * (2 + (1 if self.fp8 else 2))   # K and V: BF16 read, pool element written


def measure(kind, S, Rs, Cs, page_size, fp8, reps, launches):
    torch.manual_seed(0)
    case = Case(S, Rs, Cs, page_size, fp8)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    with torch.cuda.stream(stream):
        slot = case.slots()
        case.append(s)
        stream.synchronize()
        ours = [pool[slot].clone() for pool in (case.k_pool, case.v_pool)]
        for pool in (case.k_pool, case.v_pool):
            pool[slot] = 0
        case.recipe(s)
        stream.synchronize()
        equal = all(torch.equal(a, pool[slot]) for a, pool in zip(ours, (case.k_pool, case.v_pool)))
        case.forward(s)   # (the split workspace is sized outside the timed window)
        stream.synchronize()
    calls = {"append": case.append, "torch": case.recipe,
             "append_step": lambda s: (case.append(s), case.forward(s)),
             "torch_step": lambda s: (case.recipe(s), case.forward(s))}
    timers = {name: events_timer(lambda fn=fn: fn(s), stream, launches) for name, fn in calls.items()}
    for fn in timers.values():   # warm-up
        fn()
    us = {name: [] for name in timers}
    for _ in range(reps):
        for name, fn in timers.items():
            us[name].append(fn())
    row = {"kind": kind, "S": S, "Rs": Rs, "Cs": Cs, "Hkv": HKV, "D": D, "page_size": page_size,
           "pools": "FP8" if fp8 else "BF16", "reps": reps, "launches": launches, "bytes": case.bytes_moved(),
           "append_equals_torch": equal}
    for name, xs in us.items():
        med = statistics.median(xs)
        row[name] = {"us": round(med, 2), "us_min": round(min(xs), 2), "us_max": round(max(xs), 2)}
        if name in ("append", "torch"):
            rate = case.bytes_moved() / (med * 1e-6)
            row[name].update(tb_per_s=round(rate / 1e12, 3), of_hbm_peak=round(rate / HBM_BYTES_PER_S, 3))
    row["append_over_torch"] = round(row["append"]["us"] / row["torch"]["us"], 3)
    row["step_over_torch_step"] = round(row["append_step"]["us"] / row["torch_step"]["us"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_paged_append"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_paged_append.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "cases": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    rows = [("decode", S, 1, 4096, P_) for S in (8, 64, 256) for P_ in (16, 256)]
    rows += [("chunk", 8, 2048, 4096, P_) for P_ in (16, 256)]
    for kind, S, Rs, Cs, page_size in rows:
        for fp8 in (False, True):
            row = measure(kind, S, Rs, Cs, page_size, fp8, args.reps, args.launches)
            print(json.dumps(row), flush=True)
            result["cases"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_paged_append.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
