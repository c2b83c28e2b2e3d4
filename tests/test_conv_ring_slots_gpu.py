"""The persistent conv kernel's TMA producer passes over the ring slot the epilogue still holds, and at 112 / 128 columns half of each
staged tile lives outside the ring.  Only buffers and slot order change, so every output bit -- fp32 tensor, both fp16 planes and the
sentinels around the written channel slice -- must equal the digests recorded with the strictly round-robin ring
(tests/golden/make_golden_conv_ring_slots.py)."""
import importlib.util
import os

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_conv_ring_slots", os.path.join(HERE, "golden", "make_golden_conv_ring_slots.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _gen()


@pytest.mark.parametrize("name", sorted(GEN.CASES))
def test_conv_ring_slots_match_digests(name):
    import numpy as np
    fx = np.load(os.path.join(HERE, "golden", "conv_ring_slots.npz"))
    got = GEN.run_case(name)
    keys = sorted(k.split("/", 1)[1] for k in fx.files if k.split("/", 1)[0] == name)
    assert keys == sorted(got), (keys, sorted(got))
    for key in keys:
        assert GEN.digest(got[key]) == str(fx[f"{name}/{key}"]), f"{name}: {key} differs from the recorded output"
