"""SURVEY.md 8(f) rank 3 — test-time input pipeline (uint8 frame -> CropTop -> cv2-style bilinear Resize -> Normalize -> CHW, calibration
update): visualdet3d_b200/preprocess.py (`preprocess_host`) against fixtures generated with the unmodified reference classes
(tests/golden/make_golden_preprocess.py; strided samples, sums, the last column and the first row of every output).
Tolerance: 2e-5 on the normalised values (cv2's SIMD row / column passes may fuse multiply-adds; the bar of the path is 1e-3)."""
import os
import sys
import time

import numpy as np
import pytest

from conftest import GOLDEN
from visualdet3d_b200 import preprocess as pp

sys.path.insert(0, GOLDEN)


def _frame(seed, H, W):
    from make_golden_preprocess import frame
    return frame(seed, H, W)


def test_pipeline_matches_reference_fixtures():
    fx = np.load(os.path.join(GOLDEN, "preprocess.npz"))
    n = len([k for k in fx.files if k.endswith("_meta")])
    worst, t_tot = 0.0, 0.0
    for ci in range(n):
        seed, H, W, crop, Ho, Wo = [int(v) for v in fx[f"c{ci}_meta"]]
        for side, sd in (("l", seed), ("r", seed + 100)):
            img = _frame(sd, H, W)
            t0 = time.perf_counter()
            out = pp.preprocess_host(img, crop, (Ho, Wo))
            t_tot += time.perf_counter() - t0
            assert out.shape == (3, Ho, Wo) and out.dtype == np.float32
            st = int(fx[f"c{ci}_stride"])
            d = np.abs(out.reshape(-1)[::st] - fx[f"c{ci}_{side}_samples"]).max()
            worst = max(worst, float(d))
            assert d < 2e-5, (ci, side, d)
            if side == "l":
                assert abs(float(out.astype(np.float64).sum()) - float(fx[f"c{ci}_l_sum"])) < 1e-6 * float(fx[f"c{ci}_l_abssum"])
                assert np.abs(out[:, :, -1] - fx[f"c{ci}_last_col"]).max() < 2e-5          # right edge: cropped (cases 0-3) or zero padded then normalised (case 4)
                assert np.abs(out[:, 0, :] - fx[f"c{ci}_first_row"]).max() < 2e-5          # first row after the crop
        for nm in ("P2", "P3"):
            got = pp.adjust_calib(fx[nm], crop, H, Ho)
            assert np.array_equal(got, fx[f"c{ci}_{nm}"]), (ci, nm)                         # same float64 operations in the same order
    print(f"input pipeline: max |diff| vs the reference {worst:.2e}; host form {t_tot / (2 * n) * 1e3:.1f} ms per frame (scalar C, parity checker)")


def test_bad_arguments_are_reported():
    from visualdet3d_b200 import _lib
    with pytest.raises(_lib.Vd3dError, match="crop_top"):
        pp.preprocess_host(np.zeros((10, 20, 3), np.uint8), 12, (8, 16))        # crop_top >= H
    with pytest.raises(_lib.Vd3dError, match="bad arguments"):
        pp.preprocess_host(np.zeros((10, 20, 4), np.uint8), 2, (8, 16))         # C != 3
    with pytest.raises(_lib.Vd3dError, match="shrinks"):
        pp.preprocess_host(np.zeros((40, 20, 3), np.uint8), 0, (8, 16))         # a 5x source step: beyond the kernel's 2x stage
