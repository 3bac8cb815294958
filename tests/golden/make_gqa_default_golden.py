"""Writes tests/golden/gqa_default_outputs.json: the SHA-256 of every output of forward, dQ and dK/dV on seeded
inputs, as the library computed them before grouped K/V (FunctionConstantValues.kvGroup) existed.
tests/test_kv_group.py::test_ungrouped_results_are_unchanged checks that kvGroup 0 and 1 still produce those bits.  Every
grid is large enough (or SIMT) that no launch plan depends on the SM count.  Run on an H100 with the library to record:
    MFA_B200_LIBRARY=/path/to/libmfa_b200.so python tests/golden/make_gqa_default_golden.py"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.test_kv_group import GOLDEN, _descriptor, _inputs, run  # noqa: E402
import mfa_b200 as mfa  # noqa: E402

CASES = [dict(R=200, C=200, D=64, mode="bf16", batch=72, causal=False, seed=1),
         dict(R=130, C=257, D=128, mode="bf16", batch=70, causal=True, seed=2),
         dict(R=100, C=77, D=48, mode="fp32", batch=3, causal=True, seed=3),
         dict(R=64, C=96, D=40, mode="bf16", batch=80, causal=False, seed=4)]

out = []
for spec in CASES:
    desc = _descriptor(spec["R"], spec["C"], spec["D"], spec["mode"], batch=spec["batch"], causal=spec["causal"])
    result = run(desc, 1, _inputs(desc, 1, spec["seed"]), raw=True)
    out.append(dict(spec, sha256={k: hashlib.sha256(v.tobytes()).hexdigest() for k, v in sorted(result.items())}))
with open(GOLDEN, "w") as f:
    json.dump({"library": mfa.version(), "cases": out}, f, indent=1)
print(json.dumps(out))
