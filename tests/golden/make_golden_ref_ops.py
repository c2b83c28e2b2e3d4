"""Golden-vector generator for tests/test_dcn_iou3d_gpu.py: runs that test file on a GPU with the reference's OWN compiled DCN / iou3d
extensions (oracle/build_ref.py builds them from the reference sources into oracle/_ref) and stores what they returned (large tensors as a
fixed seeded sample) in tests/golden/ref_ops.npz; the tests then run without the reference.

    python tests/golden/make_golden_ref_ops.py [OUT.npz]
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ref_ops.npz")
    os.environ["VD3D_RECORD_REF"] = "1"
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(os.path.dirname(HERE), "test_dcn_iou3d_gpu.py")])
    rec = sys.modules["test_dcn_iou3d_gpu"].RECORD
    assert rc == 0 and rec, "the tests must pass against the reference extensions while recording"
    np.savez_compressed(out, **rec)
    print("wrote", out, len(rec), "arrays")
