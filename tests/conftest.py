import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name: str):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


@pytest.fixture(scope="session")
def golden():
    return load_golden


def pytest_sessionfinish(session, exitstatus):
    """Dump the observed parity errors recorded by the tests (ts_testutil.record_parity)."""
    try:
        import json

        import ts_testutil
        if not ts_testutil.PARITY:
            return
        out_dir = os.path.join(ROOT, "gpurun_out")
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, "parity_report.json")
        merged = {}
        if os.path.exists(path) and os.environ.get("TS_PARITY_APPEND", "0") == "1":
            merged = json.load(open(path))
        merged.update(ts_testutil.PARITY)
        with open(path, "w") as f:
            json.dump(merged, f, indent=1, sort_keys=True)
    except Exception as e:  # never turn a green run red because of the report
        sys.stderr.write(f"parity report not written: {e}\n")
