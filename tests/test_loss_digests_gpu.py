"""Every output of the five GPU training losses -- losses, terms and totals, the anchor assignment and counts, every gradient -- on every
fixture case must equal the recorded digests (tests/golden/make_golden_loss_digests.py) bit for bit.  The reference comparisons allow
1e-5, which a reordered sum passes; these do not."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_loss_digests", os.path.join(HERE, "golden", "make_golden_loss_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _gen()


@pytest.mark.parametrize("loss,case", [(loss, case) for loss, cases in GEN.CASES.items() for case in cases])
def test_loss_outputs_match_digests(loss, case):
    fx = np.load(os.path.join(HERE, "golden", "loss_digests.npz"))
    prefix = f"{loss}/{case}/"
    got = GEN.run_case(loss, case)
    keys = sorted(k[len(prefix):] for k in fx.files if k.startswith(prefix))
    assert keys == sorted(got), (keys, sorted(got))
    for key in keys:
        assert GEN.digest(got[key]) == str(fx[prefix + key]), f"{loss} {case}: {key} differs from the recorded output"
