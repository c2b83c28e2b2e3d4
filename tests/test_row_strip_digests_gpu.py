"""The row-strip kernels' outputs -- `vd3d_row_conv` fp32 and plane outputs, `vd3d_stem_pool_fused` pooled planes with and without fp32, and
the row planes of `vd3d_image_to_h16_rows` / `vd3d_image_to_h16_rows_c` -- must equal the recorded digests
(tests/golden/make_golden_row_strip_digests.py) bit for bit.  `test_row_conv_vs_fp64` allows 2e-5, which a reordered MMA chain passes;
these do not."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_row_strip_digests", os.path.join(HERE, "golden", "make_golden_row_strip_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _gen()


@pytest.mark.parametrize("case", GEN.CASES)
def test_row_strip_outputs_match_digests(case):
    fx = np.load(os.path.join(HERE, "golden", "row_strip_digests.npz"))
    prefix = f"{case}/"
    got = GEN.run_case(case)
    keys = sorted(k[len(prefix):] for k in fx.files if k.startswith(prefix))
    assert keys == sorted(set(got) - set(GEN.EXCLUDED.get(case, ()))), (keys, sorted(got))
    for key in keys:
        assert GEN.digest(got[key]) == str(fx[prefix + key]), f"{case}: {key} differs from the recorded output"
