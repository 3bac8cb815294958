"""Rotary append (mfa.appendPagedKV(..., rotary=)) against the torch recipe it replaces: device time of rotating one
step's queries and new keys by RoPE at their cache positions, writing Q in the paged forward's [H][T][D] layout and the
keys and values into shuffled page pools.  H = 32 query heads, Hkv = 8, D = 128, BF16 sources, r = 128 and 64 (NeoX
pairs), P = 16, FlashAttention-style [positions][r/2] cos / sin tables:
  decode    S = 1, 8 and 64 sequences of Rs = 1 new token over Cs = 4096 cached keys
  chunk     a chunked-prefill step: 8 sequences of 2048 new tokens (Cs = 4096)
each into BF16 pools and into FP8 E4M3 pools with per-head scales.  The recipe computes each token's position on the
device from the same tables (column_lengths[s] - Rs + i), rotates q and k op by op in float32, runs
q.transpose(0, 1).contiguous() into the forward's Q buffer, then mfa.appendPagedKV.  Each row also times a whole step:
the call followed by the split paged forward (causal, the library's plan), against the recipe followed by the same
forward.
Calls alternate after a warm-up (CUDA events, eager launches, --launches calls per timing), so that clock and thermal
drift hit both alike; each is repeated --reps times and reported as median, min and max.  Each row gives the bytes the
fused call must read and write, that rate and its share of HBM3's 3.35 TB/s, and whether its Q and pools equal the
recipe's byte for byte.  The card name and power limit are read in the same run.
Usage (on an H100):  python scripts/bench_rotary_append.py [--out-dir DIR] [--reps 5]; the JSON goes to
DIR/bench_rotary_append.json (default: a bench_rotary_append directory under the system temporary directory)."""
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
from scripts.bench_paged_append import Case, H, HKV, D, HBM_BYTES_PER_S  # noqa: E402

P = mfa.GEMMOperandPrecision


class RotaryCase(Case):
    def __init__(self, S, Rs, Cs, page_size, fp8, r):
        super().__init__(S, Rs, Cs, page_size, fp8)
        self.r = r
        self.q_new = torch.randn(self.T, H, D, device="cuda").to(torch.bfloat16)
        positions = self.page_table.shape[1] * page_size
        theta = (torch.arange(positions, device="cuda", dtype=torch.float64)[:, None] *
                 10000.0 ** (-torch.arange(0, r, 2, device="cuda", dtype=torch.float64) / r))
        self.cos, self.sin = theta.cos().float().contiguous(), theta.sin().float().contiguous()
        self.rotary = mfa.Rotary(self.q_new.data_ptr(), self.q.data_ptr(), self.cos.data_ptr(), self.sin.data_ptr(),
                                 H, 0, r, 0, positions, 0)
        self.k_rot = torch.empty_like(self.k_new)
        self.recipe_arg = mfa.PagedKVAppend(self.k_rot.data_ptr(), self.v_new.data_ptr(), self.T, 0, HKV, D,
                                            self.pool_rows, P.BF16)
        torch.cuda.synchronize()

    def fused(self, s):
        mfa.appendPagedKV(self.paged, self.append_arg, self.k_pool.data_ptr(), self.v_pool.data_ptr(),
                          fp8=self.fp8_arg, stream=s, rotary=self.rotary)

    def rope(self, x, pos):
        h = self.r // 2
        c, s = self.cos[pos][:, None, :], self.sin[pos][:, None, :]
        xf = x.float()
        a, b = xf[..., :h], xf[..., h:self.r]
        return torch.cat([a * c - b * s, b * c + a * s, xf[..., self.r:]], dim=-1).to(x.dtype)

    def recipe(self, s):
        pos = (self.lengths[self.token_seq] - self.Rs + self.token_index).long()
        self.q.copy_(self.rope(self.q_new, pos).transpose(0, 1).contiguous())
        self.k_rot.copy_(self.rope(self.k_new, pos))
        mfa.appendPagedKV(self.paged, self.recipe_arg, self.k_pool.data_ptr(), self.v_pool.data_ptr(),
                          fp8=self.fp8_arg, stream=s)

    def bytes_moved(self):
        q = self.T * H * D * 2 * 2                                     # Q read and written, BF16
        kv = 2 * self.T * HKV * D * (2 + (1 if self.fp8 else 2))       # K and V: BF16 read, pool element written
        table = self.T * self.r // 2 * 4 * 2                            # cos and sin of each token
        return q + kv + table


def measure(kind, S, Rs, Cs, page_size, fp8, r, reps, launches):
    torch.manual_seed(0)
    case = RotaryCase(S, Rs, Cs, page_size, fp8, r)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    with torch.cuda.stream(stream):
        slot = case.slots()
        case.fused(s)
        stream.synchronize()
        ours = [case.q.clone()] + [pool[slot].clone() for pool in (case.k_pool, case.v_pool)]
        case.q.zero_()
        for pool in (case.k_pool, case.v_pool):
            pool[slot] = 0
        case.recipe(s)
        stream.synchronize()
        equal = all(torch.equal(a, b) for a, b in zip(ours, [case.q] + [p[slot] for p in (case.k_pool, case.v_pool)]))
        case.forward(s)   # (the split workspace is sized outside the timed window)
        stream.synchronize()
    calls = {"fused": case.fused, "torch": case.recipe,
             "fused_step": lambda s: (case.fused(s), case.forward(s)),
             "torch_step": lambda s: (case.recipe(s), case.forward(s))}
    timers = {name: events_timer(lambda fn=fn: fn(s), stream, launches) for name, fn in calls.items()}
    for fn in timers.values():   # warm-up
        fn()
    us = {name: [] for name in timers}
    for _ in range(reps):
        for name, fn in timers.items():
            us[name].append(fn())
    row = {"kind": kind, "S": S, "Rs": Rs, "Cs": Cs, "H": H, "Hkv": HKV, "D": D, "r": r, "page_size": page_size,
           "pools": "FP8" if fp8 else "BF16", "reps": reps, "launches": launches, "bytes": case.bytes_moved(),
           "fused_equals_torch": equal}
    for name, xs in us.items():
        med = statistics.median(xs)
        row[name] = {"us": round(med, 2), "us_min": round(min(xs), 2), "us_max": round(max(xs), 2)}
        if name in ("fused", "torch"):
            rate = case.bytes_moved() / (med * 1e-6)
            row[name].update(tb_per_s=round(rate / 1e12, 3), of_hbm_peak=round(rate / HBM_BYTES_PER_S, 3))
    row["fused_over_torch"] = round(row["fused"]["us"] / row["torch"]["us"], 3)
    row["step_over_torch_step"] = round(row["fused_step"]["us"] / row["torch_step"]["us"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_rotary_append"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rotary_append.py measures on the GPU: no CUDA device")
    result = {**card(), "library": mfa.library_path(), "version": mfa.version(), "cases": []}
    print(json.dumps({k: result[k] for k in ("gpu", "power_limit", "version")}), flush=True)
    rows = [("decode", S, 1, 4096) for S in (1, 8, 64)] + [("chunk", 8, 2048, 4096)]
    for kind, S, Rs, Cs in rows:
        for r in (128, 64):
            for fp8 in (False, True):
                row = measure(kind, S, Rs, Cs, 16, fp8, r, args.reps, args.launches)
                print(json.dumps(row), flush=True)
                result["cases"].append(row)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "bench_rotary_append.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("->", path)


if __name__ == "__main__":
    main()
