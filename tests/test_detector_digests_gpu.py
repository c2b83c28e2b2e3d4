"""The six native detectors' inference outputs -- every stage-hook tensor, the kept decode rows, the counts and the launches per `launch()` --
must equal the recorded digests (tests/golden/make_golden_detector_digests.py) bit for bit.  The reference comparisons allow 1e-3, which a
reordered sum or an extra fp16 split passes; these do not."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_detector_digests", os.path.join(HERE, "golden", "make_golden_detector_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _gen()


@pytest.mark.parametrize("case", GEN.CASES)
def test_detector_outputs_match_digests(case):
    fx = np.load(os.path.join(HERE, "golden", "detector_digests.npz"))
    prefix = f"{case}/"
    got = GEN.run_case(case)
    keys = sorted(k[len(prefix):] for k in fx.files if k.startswith(prefix))
    assert keys == sorted(set(got) - set(GEN.EXCLUDED.get(case, ()))), (keys, sorted(got))
    for key in keys:
        assert np.array_equal(GEN.record(key, got[key]), fx[prefix + key]), f"{case}: {key} differs from the recorded output"
