"""The augmentation kernel (`vd3d_train_augment`), for training and as the test-time resize (`preprocess_batch`), on the constructed cases of
tests/augment_cases.py: bit for bit equal to their host forms, and within the CPU bars of the cv2 fixture (2e-6 geometry, 5e-5 colour) and of
the float64 closed forms.  Each case runs alone, then every case of one output size in a single launch (mixed source sizes, mirrors, both
warp geometries), twice with the same bits.  The output buffer is filled with NaN before each launch, so an element the kernel never writes
(a tile wholly in the pad included) fails the comparison."""
import numpy as np
import pytest
import torch

import augment_cases as ac
from conftest import GOLDEN
from visualdet3d_b200 import _lib
from visualdet3d_b200 import preprocess as pp
from visualdet3d_b200 import train_augment as ta

pytestmark = pytest.mark.gpu


def deferred(c):
    return ta.DeferredFrame(c["frame"], c["geom"], c["crop_top"], c["affine"], c["mirror"], c["ops"], c["args"], c["noise"], c["Ho"], c["Wo"],
                            ac.MEAN, ac.STD)


def launch_into_nan(frames):
    """DeferredBatch.to_device, but into an output filled with NaN first."""
    batch = ta.DeferredBatch(frames)
    B, _, Ho, Wo = batch.shape
    dev = batch.staging.to("cuda")
    descs = np.stack([f.describe(dev.data_ptr() + int(o)) for f, o in zip(frames, batch.offsets)])
    d = torch.from_numpy(descs).to("cuda")
    out = torch.full((B, 3, Ho, Wo), float("nan"), dtype=torch.float32, device="cuda")
    _lib.launch_count_reset()
    _lib.call("vd3d_train_augment", d.data_ptr(), B, 3, Ho, Wo, ta._vp(batch.mean), ta._vp(batch.std), out.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert _lib.launch_count() == 1
    return out.cpu().numpy()


def _check(cases, got, fx, worst):
    for c, g in zip(cases, got):
        host = ta.augment_host(deferred(c))
        assert np.isfinite(g).all(), (c["id"], "elements left unwritten")
        assert np.array_equal(g, host), (c["id"], float(np.abs(g - host).max()))
        d = float(np.abs(g - fx[c["id"]]).max())
        assert d <= ac.tol(c), (c["id"], d)
        want = ac.closed_form(c)
        if want is not None:
            dc = float(np.abs(g - want).max())
            assert dc <= ac.GEOMETRY_TOL, (c["id"], dc)
            d = max(d, dc)
        worst[c["group"]] = max(worst.get(c["group"], 0.0), d)


def _groups():
    by_size = {}
    for c in ac.CASES:
        by_size.setdefault((c["Ho"], c["Wo"]), []).append(c)
    return by_size


def test_each_case_alone_matches_host_bit_for_bit():
    fx = np.load(f"{GOLDEN}/augment_cases.npz")
    worst = {}
    for c in ac.CASES:
        _check([c], launch_into_nan([deferred(c)]), fx, worst)
    print("kernel alone vs fixture / closed forms, max |diff| per group: " + ", ".join(f"{g} {d:.2e}" for g, d in worst.items()))


def test_one_launch_per_output_size_twice():
    fx = np.load(f"{GOLDEN}/augment_cases.npz")
    worst = {}
    mixed = 0
    for (Ho, Wo), cases in _groups().items():
        frames = [deferred(c) for c in cases]
        first = launch_into_nan(frames)
        _check(cases, first, fx, worst)
        assert np.array_equal(first, launch_into_nan(frames))               # same bits on a second launch
        assert torch.equal(torch.from_numpy(first), ta.augment_batch(frames, "cuda").cpu())     # the product path too
        if len({c["frame"].shape for c in cases}) > 1 and len({c["mirror"] for c in cases}) > 1:
            mixed += 1
    assert mixed >= 1
    print("kernel batched by output size vs fixture / closed forms, max |diff| per group: "
          + ", ".join(f"{g} {d:.2e}" for g, d in worst.items()))


def test_preprocess_kernel_on_resize_cases():
    """The test-time resize has no mirror: a mirrored case's frame gives the closed form of its unmirrored twin."""
    worst = 0.0
    groups = {}
    for c in ac.CASES:
        if c["geom"] == ac.GEOM_RESIZE and len(c["ops"]) == 0:
            groups.setdefault((c["crop_top"], c["Ho"], c["Wo"]), []).append(c)
    for (crop, Ho, Wo), cases in groups.items():
        frames = [c["frame"] for c in cases]
        for batch in [[f] for f in frames] + ([frames] if len(frames) > 1 else []):
            got = pp.preprocess_batch(batch, crop, (Ho, Wo), ac.MEAN, ac.STD, device="cuda").cpu().numpy()
            for f, g in zip(batch, got):
                c = cases[next(i for i, x in enumerate(frames) if x is f)]
                assert np.array_equal(g, pp.preprocess_host(f, crop, (Ho, Wo), ac.MEAN, ac.STD)), c["id"]
                want = ac.closed_form(dict(c, mirror=0))
                d = float(np.abs(g - want).max())
                worst = max(worst, d)
                assert d <= ac.GEOMETRY_TOL, (c["id"], d)
    print(f"preprocess kernel vs closed forms on the resize cases: max |diff| {worst:.2e}")
