"""Measured parity of the CUDA path against the CPU oracle at the BASELINE.json configs, one JSON line per
(config, dtype policy, output): max-abs, max-rel and relative RMS error.

  max_rel = max |a - b| / max(|b|, 1e-3 * rms(b))
  rel_rms = rms(a - b) / rms(b)

The oracle (oracle/network_oracle.c, the C restatement of the reference's Network.swift) runs on the inputs AFTER
rounding to the kernel's memory format, so the numbers isolate the kernel's own arithmetic.  `vs_f64` repeats the
comparison against the float64 matrix-form implementation (oracle/oracle_np.py) as a tie-breaker: where the FP32
oracle itself carries summation error (N = 4096+), `vs_f64` is the cleaner figure.

Usage (GPU box):  python scripts/parity_table.py [--out gpurun_out/parity.jsonl] [--quick]
TEST INFRASTRUCTURE: imports oracle/ as the checker, like tests/.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def error_stats(actual, expected):
    a, b = np.asarray(actual, np.float64), np.asarray(expected, np.float64)
    err = np.abs(a - b)
    rms_b = float(np.sqrt(np.mean(b * b)))
    floor = max(1e-3 * rms_b, 1e-30)
    return {"max_abs": float(err.max()), "max_rel": float((err / np.maximum(np.abs(b), floor)).max()),
            "rel_rms": float(np.sqrt(np.mean(err * err)) / max(rms_b, 1e-30)), "rms_ref": rms_b}


def run_config(name, R, C, D, policy, backward, seed, threads, lowMid=False, f64=True, transpose=(False,) * 4):
    import mfa_b200 as mfa
    import oracle
    from oracle.oracle_np import attention_f64
    from tests.attention_harness import run_attention, oracle_outputs

    P = mfa.GEMMOperandPrecision
    desc = mfa.AttentionDescriptor()
    desc.lowPrecisionInputs = policy != "fp32"
    desc.lowPrecisionIntermediates = lowMid
    desc.matrixDimensions = (R, C, D)
    desc.transposeState = tuple(transpose)
    if policy == "bf16":
        desc.inputPrecisionOverride = P.BF16
    elif policy == "fp16":
        desc.inputPrecisionOverride = P.FP16
    # policy == "reference": FP16 Q/K/V + BF16 dO (AttentionDescriptor+Precisions.swift:13-23)
    prec = desc.memoryPrecisions
    Op, KT = mfa.AttentionOperand, mfa.AttentionKernelType
    net = oracle.Network(R, C, D, seed=seed, threads=threads)
    if policy != "fp32":
        net.round_inputs(int(prec[Op.Q]), int(prec[Op.dO]))
    types = list(KT) if backward else [KT.forward]
    backends = {t.name: desc.kernelDescriptor(t).backend.name for t in types}
    t0 = time.perf_counter()
    out = run_attention(desc, net, types=types)
    t_gpu = time.perf_counter() - t0
    t0 = time.perf_counter()
    ref = oracle_outputs(net, backward=backward)
    t_cpu = time.perf_counter() - t0
    ref64 = attention_f64(net.Q, net.K, net.V, net.dO if backward else None) if f64 else None
    rows = []
    for key in (("O", "L", "D", "dQ", "dK", "dV") if backward else ("O", "L")):
        row = {"config": name, "R": R, "C": C, "D": D, "policy": policy, "lowPrecisionIntermediates": lowMid,
               "output": key, "backend": backends, **error_stats(out[key], ref[key])}
        if ref64 is not None:
            s = error_stats(out[key], ref64[key])
            row["vs_f64"] = {k: s[k] for k in ("max_abs", "max_rel", "rel_rms")}
            s = error_stats(ref[key], ref64[key])
            row["oracle_vs_f64_rel_rms"] = s["rel_rms"]
        row["oracle_s"], row["gpu_call_s"] = round(t_cpu, 2), round(t_gpu, 2)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("gpurun_out", "parity.jsonl"))
    ap.add_argument("--quick", action="store_true", help="skip the N=8192 D=256 oracle run")
    args = ap.parse_args()
    import oracle
    threads = min(oracle.max_threads(), len(os.sched_getaffinity(0)))
    configs = [
        ("config2 fwd N=4096 D=128", 4096, 4096, 128, "bf16", False, 0),
        ("config2 fwd N=4096 D=128", 4096, 4096, 128, "fp16", False, 0),
        ("config3 fwd+bwd N=2048 D=64", 2048, 2048, 64, "reference", True, 2),
        ("config3 fwd+bwd N=2048 D=64", 2048, 2048, 64, "fp16", True, 0),
        ("config3 fwd+bwd N=2048 D=64", 2048, 2048, 64, "bf16", True, 1),
        ("fwd+bwd N=4096 D=128", 4096, 4096, 128, "bf16", True, 3),
        ("fwd+bwd N=4096 D=128", 4096, 4096, 128, "fp16", True, 3),
        ("fwd+bwd N=2048 D=256", 2048, 2048, 256, "bf16", True, 5),
        ("fwd+bwd N=1000 D=72 ragged", 1000, 777, 72, "reference", True, 6),
        ("fwd+bwd N=2048 D=256 reference", 2048, 2048, 256, "reference", True, 8),
        ("fwd+bwd N=2048 D=128 Q,K,V,O transposed", 2048, 2048, 128, "fp16", True, 9),
        ("fwd+bwd N=1024 D=64 K,O transposed", 1024, 1536, 64, "bf16", True, 10),
        ("config1 fwd+bwd N=128 D=64 fp32", 128, 128, 64, "fp32", True, 7),
    ]
    if not args.quick:
        configs.append(("config4 fwd N=8192 D=256", 8192, 8192, 256, "bf16", False, 4))
        configs.append(("config4 fwd N=8192 D=256", 8192, 8192, 256, "fp16", False, 4))
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        for name, R, C, D, policy, backward, seed in configs:
            try:
                transpose = (True,) * 4 if "Q,K,V,O transposed" in name else ((False, True, False, True) if "K,O transposed" in name
                                                                              else (False,) * 4)
                rows = run_config(name, R, C, D, policy, backward, seed, threads, f64=R <= 4096, transpose=transpose)
            except Exception as exc:  # keep going: a failing config is a row in the table too
                rows = [{"config": name, "policy": policy, "error": repr(exc)}]
            for row in rows:
                f.write(json.dumps(row) + "\n")
                f.flush()
                if "error" in row:
                    print(row)
                else:
                    print(f"{row['config']:34s} {row['policy']:9s} {row['output']:2s} max_abs {row['max_abs']:.3e} "
                          f"max_rel {row['max_rel']:.3e} rel_rms {row['rel_rms']:.3e}"
                          + (f"  | vs f64 rel_rms {row['vs_f64']['rel_rms']:.3e}" if "vs_f64" in row else ""),
                          flush=True)


if __name__ == "__main__":
    main()
