import glob
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    # GPU tests are selected with `-m gpu`; when no device is visible they are skipped
    # rather than failed so that a plain `pytest tests/` works on the CPU box.
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """Fixtures produced by the reference itself (tests/golden/make_golden.py)."""

    def __init__(self):
        g = os.path.join(ROOT, "tests", "golden")
        with open(os.path.join(g, "golden_v1.json")) as fh:
            self.meta = json.load(fh)
        # the arrays are stored in parts below 1 MB each (golden_v1_00.npz, ...; make_golden.save_parts)
        self.arr = {}
        for part in sorted(glob.glob(os.path.join(g, "golden_v1_*.npz"))):
            with np.load(part) as z:
                self.arr.update((k, z[k]) for k in z.files)
        self.cases = self.meta["cases"]

    def get(self, case, key):
        return self.arr[f"{case['name']}__{key}"]

    def has(self, case, key):
        return f"{case['name']}__{key}" in self.arr


_golden = None


def golden():
    global _golden
    if _golden is None:
        _golden = Golden()
    return _golden


@pytest.fixture(scope="session")
def gold():
    return golden()
