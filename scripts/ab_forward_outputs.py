"""O and L of the bf16 forward on seeded inputs, for comparing two builds of the library output for output.

    MFA_B200_LIBRARY=/path/to/old/libmfa_b200.so python scripts/ab_forward_outputs.py --out DIR_A
    python scripts/ab_forward_outputs.py --out DIR_B
    python scripts/ab_forward_outputs.py --compare DIR_A DIR_B      # exit status 1 unless every array is bitwise equal

Shapes: causal 4096 x 4096 (64 heads), one head of N = 4096 (a split-KV grid and the merge), D = 64 and D = 256 at
N = 8192, and a ragged shape (rows and keys not multiples of the tiles, D short of its 128 columns).  Then every other
call form of the forward at D = 64, 128 and 256 (CASES): packed sequences, a paged cache, sliding windows on fixed,
packed and paged calls, split packed and paged decode steps whose plan packs a K/V group's query heads into one tile and
cuts the keys into several ranges, and FP8 pools unsplit and split.  O is written in full, in FP32; L as the kernel
stores it (log2 units).  Each entry of shapes.json records the call's launch count (and for split calls its plan)."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (R, C, D, heads, causal)
SHAPES = {
    "causal_4096_d128_h64": (4096, 4096, 128, 64, True),
    "single_head_split_4096_d128": (4096, 4096, 128, 1, False),
    "n8192_d64_h8": (8192, 8192, 64, 8, False),
    "n8192_d256_h8": (8192, 8192, 256, 8, False),
    "ragged_1000x1500_d120_h3": (1000, 1500, 120, 3, False),
}

# name: (form, D, causal, window, split num_splits or None, fp8): packed and paged calls over S sequences of ragged
# lengths, H = 8 query heads on H / G K/V heads; the split decode steps have 3 queries per sequence and G = 4
CASES = {}
for _D in (64, 128, 256):
    CASES.update({
        f"packed_d{_D}": ("packed", _D, False, None, None, False),
        f"paged_d{_D}": ("paged", _D, True, None, None, False),
        f"window_fixed_d{_D}": ("fixed", _D, False, (200, 50), None, False),
        f"window_packed_d{_D}": ("packed", _D, True, (100, 0), None, False),
        f"window_paged_d{_D}": ("paged", _D, True, (150, 0), None, False),
        f"split_packed_d{_D}": ("packed_decode", _D, True, None, 3, False),
        f"split_paged_d{_D}": ("paged_decode", _D, True, None, 3, False),
        f"fp8_paged_d{_D}": ("paged", _D, True, None, None, True),
        f"fp8_split_paged_d{_D}": ("paged_decode", _D, True, None, 3, True),
    })


def run_case(mfa, torch, seed, form, D, causal, window, num_splits, fp8):
    """O, L and the launch record of one call of CASES"""
    Op, H = mfa.AttentionOperand, 8
    G = 4 if form.endswith("decode") else 2
    decode = form.endswith("decode")
    gen = torch.Generator(device="cuda").manual_seed(seed)
    S = 5 if decode else 3
    rows = [3] * S if decode else [40, 130, 7][:S]
    keys = [700, 333, 1, 512, 129][:S] if decode else [300, 257, 90][:S]
    T = sum(rows)
    row_offsets = torch.tensor([0] + list(np.cumsum(rows)), dtype=torch.int32, device="cuda")
    q = torch.randn(H, T, D, device="cuda", generator=gen).to(torch.bfloat16)
    O = torch.full((H, T, D), float("nan"), device="cuda")
    L = torch.full((H, T), float("nan"), device="cuda")
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = True
    desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16
    desc.transposeState = (False,) * 4
    desc.batchCount = H
    desc.causal = causal
    constants = mfa.FunctionConstantValues()
    table = {}
    if form == "fixed":
        R = C = 1000
        q = torch.randn(H, R, D, device="cuda", generator=gen).to(torch.bfloat16)
        k, v = (torch.randn(H, C, D, device="cuda", generator=gen).to(torch.bfloat16) for _ in range(2))
        O = torch.full((H, R, D), float("nan"), device="cuda")
        L = torch.full((H, R), float("nan"), device="cuda")
        desc.matrixDimensions = (R, C, D)
        desc.setFunctionConstants(constants)
    elif form.startswith("packed"):
        Tk = sum(keys)
        column_offsets = torch.tensor([0] + list(np.cumsum(keys)), dtype=torch.int32, device="cuda")
        k, v = (torch.randn(H // G, Tk, D, device="cuda", generator=gen).to(torch.bfloat16) for _ in range(2))
        desc.matrixDimensions = (T, Tk, D)
        desc.setFunctionConstants(constants)
        table["sequences"] = mfa.SequenceTable(S, max(rows), max(keys), row_offsets.data_ptr(),
                                               column_offsets.data_ptr())
    else:
        P = 64 if decode else 16
        per_seq = max(-(-c // P) for c in keys)
        pages = S * per_seq + 4
        page_table = torch.randperm(pages, device="cuda", generator=gen)[:S * per_seq].view(S, per_seq).to(torch.int32)
        lengths = torch.tensor(keys, dtype=torch.int32, device="cuda")
        pools = [torch.randn(pages * P, H // G, D, device="cuda", generator=gen) for _ in range(2)]
        if fp8:
            k, v = ((p * 4).to(torch.float8_e4m3fn).view(torch.uint8) for p in pools)
            table["fp8"] = mfa.FP8KV()
        else:
            k, v = (p.to(torch.bfloat16) for p in pools)
        desc.matrixDimensions = (T, pages * P, D)
        desc.setFunctionConstants(constants)
        constants._c.kv_group = G
        table["paged"] = mfa.PagedKV(S, max(rows), row_offsets.data_ptr(), lengths.data_ptr(), page_table.data_ptr(),
                                     per_seq, P)
    if form.startswith("packed"):
        constants._c.kv_group = G
    kernel = mfa.AttentionKernel(desc.kernelDescriptor(mfa.AttentionKernelType.forward), window=window)
    tables = {key: table[key] for key in ("sequences", "paged") if key in table}
    if num_splits is not None:
        split = mfa.SplitKV(num_splits)
        plan = kernel.splitPlan(constants, split=split, **tables)
        record = {"splits": plan.splits, "heads_per_tile": plan.heads_per_tile, "grid": plan.grid_size,
                  "launches": plan.launch_count}
        table["split"] = split
    else:
        record = {"grid": kernel.gridSize(constants, **tables), "launches": kernel.launchCount(constants, **tables)}
    kernel.encode(constants, {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(),
                              Op.L: L.data_ptr()}, **table)
    torch.cuda.synchronize()
    return O.cpu().numpy(), L.cpu().numpy(), record


def dump(out_dir):
    import torch
    import mfa_b200 as mfa
    Op = mfa.AttentionOperand
    os.makedirs(out_dir, exist_ok=True)
    info = {"library": mfa.library_path(), "version": mfa.version(), "shapes": {}}
    for i, (name, (R, C, D, H, causal)) in enumerate(SHAPES.items()):
        desc = mfa.AttentionDescriptor()
        desc.lowPrecisionInputs = True
        desc.inputPrecisionOverride = mfa.GEMMOperandPrecision.BF16
        desc.matrixDimensions = (R, C, D)
        desc.transposeState = (False,) * 4
        desc.batchCount = H
        desc.causal = causal
        constants = mfa.FunctionConstantValues()
        desc.setFunctionConstants(constants)
        kernel = mfa.AttentionKernel(desc.kernelDescriptor(mfa.AttentionKernelType.forward))
        gen = torch.Generator(device="cuda").manual_seed(1000 + i)
        q = torch.randn(H, R, D, device="cuda", generator=gen).to(torch.bfloat16)
        k, v = (torch.randn(H, C, D, device="cuda", generator=gen).to(torch.bfloat16) for _ in range(2))
        O = torch.full((H, R, D), float("nan"), device="cuda")
        L = torch.full((H, R), float("nan"), device="cuda")
        kernel.encode(constants, {Op.Q: q.data_ptr(), Op.K: k.data_ptr(), Op.V: v.data_ptr(), Op.O: O.data_ptr(),
                                  Op.L: L.data_ptr()})
        torch.cuda.synchronize()
        np.save(os.path.join(out_dir, f"{name}_O.npy"), O.cpu().numpy())
        np.save(os.path.join(out_dir, f"{name}_L.npy"), L.cpu().numpy())
        info["shapes"][name] = {"R": R, "C": C, "D": D, "heads": H, "causal": causal,
                                "launches": kernel.launchCount(constants)}
    for i, (name, case) in enumerate(CASES.items()):
        O, L, record = run_case(mfa, torch, 2000 + i, *case)
        np.save(os.path.join(out_dir, f"{name}_O.npy"), O)
        np.save(os.path.join(out_dir, f"{name}_L.npy"), L)
        info["shapes"][name] = record
    with open(os.path.join(out_dir, "shapes.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


def compare(a, b):
    ok = True
    records = []
    for d in (a, b):
        with open(os.path.join(d, "shapes.json")) as f:
            records.append(json.load(f)["shapes"])
    for name in list(SHAPES) + list(CASES):
        same = records[0].get(name) == records[1].get(name)
        print(f"{name} launches: {'identical' if same else f'DIFFERENT {records[0].get(name)} -> {records[1].get(name)}'}")
        ok &= same
        for out in ("O", "L"):
            x, y = (np.load(os.path.join(d, f"{name}_{out}.npy")) for d in (a, b))
            same = x.shape == y.shape and np.array_equal(x, y, equal_nan=True)
            diff = 0.0 if same or x.shape != y.shape else float(np.nanmax(np.abs(x.astype(np.float64) - y)))
            print(f"{name} {out}: {'identical' if same else f'DIFFERENT (max |diff| {diff:.3e})'}")
            ok &= same
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory to write the arrays to")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    if not args.out:
        ap.error("--out or --compare is required")
    dump(args.out)


if __name__ == "__main__":
    main()
