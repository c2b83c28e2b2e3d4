"""The test-time input pipeline's host form (`preprocess.preprocess_host`) bit for bit against the SHA-256 digests of
tests/golden/make_golden_preprocess_digests.py: the preprocess.npz frames, every plain-resize case of tests/augment_cases.py and the bench.py
geometries."""
import sys

import numpy as np

from conftest import GOLDEN
from visualdet3d_b200 import preprocess as pp

sys.path.insert(0, GOLDEN)
from make_golden_preprocess_digests import OUT, cases, digest  # noqa: E402


def test_host_form_matches_digests():
    fx = np.load(OUT)
    cs = cases()
    assert sorted(c["id"] for c in cs) == sorted(fx.files)
    for c in cs:
        got = pp.preprocess_host(c["frame"], c["crop_top"], c["size"], c["mean"], c["std"])
        assert got.shape == (3, *c["size"]) and got.dtype == np.float32
        assert digest(got) == str(fx[c["id"]]), c["id"]
