"""O and L of the bf16 forward on seeded inputs, for comparing two builds of the library output for output.

    MFA_B200_LIBRARY=/path/to/old/libmfa_b200.so python scripts/ab_forward_outputs.py --out DIR_A
    python scripts/ab_forward_outputs.py --out DIR_B
    python scripts/ab_forward_outputs.py --compare DIR_A DIR_B      # exit status 1 unless every array is bitwise equal

Shapes: causal 4096 x 4096 (64 heads), one head of N = 4096 (a split-KV grid and the merge), D = 64 and D = 256 at
N = 8192, and a ragged shape (rows and keys not multiples of the tiles, D short of its 128 columns).  O is written in
full, in FP32; L as the kernel stores it (log2 units)."""
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
    with open(os.path.join(out_dir, "shapes.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


def compare(a, b):
    ok = True
    for name in SHAPES:
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
