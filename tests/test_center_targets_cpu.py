"""Host form of the KM3D / MonoFlex target encoder (visualdet3d_b200/center_targets.py:build_targets_host, csrc/center_targets.cu) against
the unmodified reference `_build_target` of both datasets (tests/golden/center_targets.npz, tests/golden/make_golden_center_targets.py).
Heatmaps, every integer and mask target and edge_indices are bit-exact; float targets agree within 1e-5.  The exception is the targets
measured from a projected keypoint or centre (hps, hp_offset, reg): the projector's atan2 / sin / cos may round an ulp away from torch's
CPU kernels, which moves the keypoint by an ulp of its heatmap coordinate (3.1e-5 at x = 300), so those agree within 2 ulps of the
coordinate they were measured from.  The fixtures keep every such coordinate 1e-3 px from an integer, so no index can change."""
import types

import numpy as np
import pytest

from conftest import load_fixture
from visualdet3d_b200 import _lib
from visualdet3d_b200 import center_targets as ct

FX = load_fixture("center_targets")
CASES = [f"c{i}" for i in range(int(FX["n_cases"]))]


def _labels(c):
    return [types.SimpleNamespace(**dict(zip(("x", "y", "z", "w", "h", "l", "ry", "bbox_l", "bbox_t", "bbox_r", "bbox_b"), row)))
            for row in c["objs"]]


def targets(c):
    return {k[2:]: v for k, v in c.items() if k.startswith("t/")}


def deferred(c):
    H, W = (int(v) for v in c["hw"])
    return ct.DeferredTargets.build((H, W, 3), c["P2"], _labels(c), c["cls"], 3, int(c["mode"]))


PROJECTED = ("hps", "hp_offset", "reg")


def float_close(key, got, want, hm_w):
    tol = 1e-5
    if key in PROJECTED:                               # |coordinate| <= |target| + hm_w: the target minus an integer in [0, hm_w)
        tol = np.maximum(tol, 2 * np.spacing(np.abs(want) + np.float32(hm_w)))
    return np.abs(got.astype(np.float64) - want) <= tol


@pytest.mark.parametrize("case", CASES)
def test_host_form_matches_reference(case):
    c = FX[case]
    if int(c["raises"]):
        with pytest.raises(IndexError):
            deferred(c)
        return
    got = ct.build_targets_host(deferred(c))
    assert list(got) == [str(k) for k in c["keys"]]                     # the reference's keys, in its order
    worst = 0.0
    for key, want in targets(c).items():
        g = got[key]
        assert g.dtype == want.dtype and g.shape == want.shape, (key, g.dtype, want.dtype, g.shape, want.shape)
        if key in ("hm", "hm_hp") or want.dtype != np.float32:
            assert np.array_equal(g, want), key
        else:
            ok = float_close(key, g, want, int(c["hw"][1]) // 4)
            assert ok.all(), (key, np.argwhere(~ok)[:4], g[~ok][:4], want[~ok][:4])
            worst = max(worst, float(np.abs(g.astype(np.float64) - want).max(initial=0.0)))
    print(f"{c['name']} (mode {int(c['mode'])}): float targets max |diff| {worst:.2e}")


def test_heatmaps_are_not_trivial():
    """The fixtures exercise the render: peaks of 1 and Gaussian tails in both heatmaps of both detectors."""
    for mode in (0, 1):
        hm = [FX[k]["t/hm"] for k in CASES if int(FX[k]["mode"]) == mode and not int(FX[k]["raises"])]
        hp = [FX[k]["t/hm_hp"] for k in CASES if int(FX[k]["mode"]) == mode and not int(FX[k]["raises"])]
        for maps in (hm, hp):
            v = np.concatenate([m.reshape(-1) for m in maps])
            assert (v == 1).sum() > 10 and ((v > 0) & (v < 1)).sum() > 1000


@pytest.mark.parametrize("H,W", [(384, 1280), (375, 1242), (96, 320), (4, 4)])
def test_edge_indices_formula(H, W):
    x_max, y_max = H // 4, W // 4
    e = ct.edge_indices(H, W)
    assert e.dtype == np.int64 and e.ndim == 2 and e.shape[1] == 2
    assert len(e) == 2 * (x_max + y_max)                               # the border once, corners included
    assert np.array_equal(e, np.unique(e, axis=0))
    assert set(map(tuple, e)) == {(x, y) for x in range(x_max + 1) for y in range(y_max + 1) if x in (0, x_max) or y in (0, y_max)}


def test_more_than_32_objects_raise_before_packing():
    c = FX["c0"]
    labels = _labels(FX[next(k for k in CASES if FX[k]["objs"].shape[0] == 32)]) * 2
    with pytest.raises(IndexError):
        ct.DeferredTargets.build((384, 1280, 3), c["P2"], labels[:33], [0] * 33, 3, ct.MODE_KM3D)


def _host(rec, mode, H, W, C):
    outs = {key: np.zeros(shape, dt) for key, dt, shape in ct._shapes(mode, C, H, W)}
    ptrs = (ct.ctypes.c_void_p * len(ct._SLOTS))(*[outs[key].ctypes.data for key, _, _ in ct._SLOTS])
    _lib.call("vd3d_center_targets_host", ct._vp(rec), mode, H, W, C, ptrs)


def test_malformed_records_are_rejected():
    t = deferred(FX[next(k for k in CASES if FX[k]["objs"].shape[0] == 6)])
    rb = t.record.view(np.int32)
    n_at = rb.size - 6                                                 # n, mode, img_h, img_w, num_classes, pad close the record
    assert rb[n_at] == 6 and rb[n_at + 1] == t.mode and rb[n_at + 2] == t.img_h
    _host(t.record, t.mode, t.img_h, t.img_w, 3)                       # the well-formed record runs
    bad = {"33 objects": (n_at, 33), "negative count": (n_at, -1), "class out of range": (n_at - 32, 3),
           "negative class": (n_at - 32, -1)}
    for what, (i, v) in bad.items():
        r = t.record.copy()
        r.view(np.int32)[i] = v
        with pytest.raises(_lib.Vd3dError):
            _host(r, t.mode, t.img_h, t.img_w, 3)
    with pytest.raises(_lib.Vd3dError):                                # record made for another detector / size / class count
        _host(t.record, 1 - t.mode, t.img_h, t.img_w, 3)
    with pytest.raises(_lib.Vd3dError):
        _host(t.record, t.mode, t.img_h, t.img_w + 4, 3)
    with pytest.raises(_lib.Vd3dError):
        _host(t.record, t.mode, t.img_h, t.img_w, 4)
    objs = np.zeros((1, 11))
    P2 = FX["c0"]["P2"]
    for args in ((2, 384, 1280, 3, P2, 1, objs, [0]), (0, 2, 1280, 3, P2, 1, objs, [0]), (0, 384, 1280, 0, P2, 1, objs, [0]),
                 (0, 384, 1280, 3, P2, 1, objs, [3]), (0, 384, 1280, 3, P2, 1, objs + np.nan, [0]), (0, 384, 1280, 3, P2 * 0, 1, objs, [0])):
        rec = np.zeros(t.record.size, np.uint8)
        mode, H, W, C, p2, n, o, cls = args
        with pytest.raises(_lib.Vd3dError):
            _lib.call("vd3d_center_targets_pack", ct._vp(rec), mode, H, W, C, ct._vp(np.ascontiguousarray(p2, np.float64)), n,
                      ct._vp(np.ascontiguousarray(o, np.float64)), ct._vp(np.array(cls, np.int32)))
