import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on the GPU box)")


@pytest.fixture(scope="session", autouse=True)
def _native_built():
    """The CPU suite also needs libmfa_b200.so (symbol/ABI checks) and liboracle.so."""
    lib = os.path.join(ROOT, "metal-flash-attention_b200", "lib", "libmfa_b200.so")
    ora = os.path.join(ROOT, "oracle", "_build", "liboracle.so")
    if not (os.path.exists(lib) and os.path.exists(ora)):
        import __graft_entry__
        __graft_entry__.build()


def pytest_sessionfinish(session, exitstatus):
    """Dump the measured error of every harness check of this session (GPU runs) to gpurun_out/parity_tests.jsonl."""
    import json
    harness = sys.modules.get("tests.attention_harness")
    if harness is None or not harness.RECORDS:
        return
    out = os.path.join(ROOT, "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "parity_tests.jsonl"), "w") as f:
        for row in harness.RECORDS:
            f.write(json.dumps(row) + "\n")
