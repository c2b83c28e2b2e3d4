import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100; select with -m gpu)")


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


def load_fixture(name):
    """npz fixture -> nested dict (keys 'a/b' are regrouped)."""
    import numpy as np
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    out = {}
    for k in z.files:
        if "/" in k:
            a, b = k.split("/", 1)
            out.setdefault(a, {})[b] = z[k]
        else:
            out[k] = z[k]
    return out


def subsample_like(t, fx):
    """Strided samples of tensor t matching fixture entry fx (see tests/golden/make_golden.py::subsample)."""
    import torch
    f = t.detach().reshape(-1).to(torch.float64).cpu()
    assert list(t.shape) == fx["shape"].tolist(), (list(t.shape), fx["shape"].tolist())
    return f[:: int(fx["stride"])].to(torch.float32).numpy()
