import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def rel_err(a, ref):
    """max|a - ref| / max|ref| -- the parity metric of SURVEY.md 8c (per tensor)."""
    a = np.asarray(a, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    denom = max(float(np.abs(ref).max()), 1e-30)
    return float(np.abs(a - ref).max()) / denom


class GoldenRecord:
    """One golden record: `name.npz` merged with its `name.partN.npz` parts (tests/golden/golden_io.py)."""

    def __init__(self, name):
        stem = name[:-4]
        paths = [os.path.join(GOLDEN, name)]
        i = 1
        while os.path.isfile(os.path.join(GOLDEN, "%s.part%d.npz" % (stem, i))):
            paths.append(os.path.join(GOLDEN, "%s.part%d.npz" % (stem, i)))
            i += 1
        self._arrays = {}
        for p in paths:
            with np.load(p, allow_pickle=False) as z:
                self._arrays.update({k: z[k] for k in z.files})
        self.files = list(self._arrays)

    def __getitem__(self, key):
        return self._arrays[key]

    def __contains__(self, key):
        return key in self._arrays


@pytest.fixture(scope="session")
def golden():
    return GoldenRecord
