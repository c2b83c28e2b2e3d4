"""CPU-side checks of the native disparity loss (visualdet3d_b200/disparity_loss.py): the fixture's inputs regenerate from their seeds, the
float64 restatement the kernels implement agrees with the unmodified reference's fixture values (the [max_disp - 1, max_disp) band
included), every refusal raises before the library is loaded, and the opt-in installer rebinds only DisparityLoss.forward."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_fixture
from visualdet3d_b200 import _lib, disparity_loss

FX = load_fixture("disparity_loss")
CASES = ["a", "b", "c", "d"]


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_disparity_loss", os.path.join(GOLDEN, "make_golden_disparity_loss.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = golden_module()


@pytest.mark.parametrize("case", CASES)
def test_inputs_regenerate_from_seeds(case):
    fx = FX[case]
    x, label = GEN.inputs(case)
    assert tuple(x.shape) == tuple(int(fx[k]) for k in ("B", "D", "H", "W"))
    assert GEN.sha(x) == str(fx["x_sha"]) and GEN.sha(label) == str(fx["label_sha"])
    D = int(fx["max_disp"])
    assert int(((label > 0) & (label < D)).sum()) == int(fx["outer_count"])


def test_fixture_covers_the_edges():
    a, b, c, d = (FX[k] for k in CASES)
    assert 0.18 < int(a["outer_count"]) / (4 * 72 * 320) < 0.28             # about 23 % valid at the training shape
    _, la = GEN.inputs("a")
    assert float(la.max()) > 96 and ((la >= 95) & (la < 96)).any()
    assert int(c["outer_count"]) == 0 and float(c["loss"]) == 0 and float(c["grad_max"]) == 0
    _, lb = GEN.inputs("b")
    assert not ((lb[0] > 0) & (lb[0] < 96)).any()                            # an image with no valid pixel
    assert len(b["named"]) >= 11 and len(a["named"]) > 0 and len(d["named"]) > 0


@pytest.mark.parametrize("case", CASES)
def test_restatement_matches_reference_fixture(case):
    """Pins the formulas csrc/disparity_loss.cu implements: loss within 1e-6 relative, gradient within 1e-6 of its max."""
    fx = FX[case]
    x, label = GEN.inputs(case)
    loss, grad, gmax = GEN.restate(x, label, int(fx["max_disp"]), fx["grad_idx"])
    ref = float(fx["loss"])
    assert abs(loss - ref) <= 1e-6 * abs(ref), (loss, ref)
    assert abs(loss - float(fx["loss64"])) <= 1e-12 * max(abs(loss), 1e-30)
    scale = max(float(fx["grad_max"]), 1e-30)
    assert np.abs(grad - fx["grad"].astype(np.float64)).max() <= 1e-6 * scale
    assert abs(gmax - float(fx["grad_max"])) <= 1e-6 * scale
    # pixels of the band [max_disp - 1, max_disp): inside the loss mask, outside the target's -- a 1e-40 target, a negligible gradient
    D, H, W = (int(fx[k]) for k in ("D", "H", "W"))
    for b, y, xx in fx["named"]:
        if not D - 1 <= float(label[b, y, xx]) < D:
            continue
        sel = np.isin(fx["grad_idx"], ((b * D + np.arange(D)) * H + y) * W + xx)
        assert sel.sum() == D
        assert np.abs(fx["grad"][sel]).max() <= 1e-30 and np.abs(grad[sel]).max() <= 1e-30


class _Crit:
    def __init__(self, **kw):
        self.max_disp, self.start_disp, self.dilation, self.weights, self.focal_coefficient = 96, 0, 1, None, 0.0
        self.__dict__.update(kw)


class _Loss:
    def __init__(self, **kw):
        self.criterion = _Crit(**kw)


def test_refusals_raise_before_the_library_loads(monkeypatch):
    def no_load():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_load)
    x, lab = torch.zeros(2, 96, 4, 8), torch.ones(2, 4, 8)

    def refused(exc, match, *args, **kw):
        with pytest.raises(exc, match=match):
            disparity_loss.disparity_loss(*args, **kw)
    refused(RuntimeError, "CUDA", x, lab)                                    # no CPU path
    refused(RuntimeError, "float32", x.double(), lab)
    refused(RuntimeError, "float32", x, lab.half())
    refused(ValueError, "max_disp", x, lab, 64)                              # D != max_disp
    refused(ValueError, "does not match", x, lab[:, :3])                     # a label at another H, W (the rescale branch)
    refused(ValueError, "does not match", x, lab[:1])
    refused(ValueError, "multi-level", [x, x], lab)
    refused(ValueError, r"\[B, max_disp, H, W\]", x[0], lab)
    refused(RuntimeError, "CUDA", x, lab[:, None])                           # a [B, 1, H, W] label passes the shape checks
    for kw, match in ((dict(focal_coefficient=1.0), "focal_coefficient"), (dict(start_disp=2), "start_disp"),
                      (dict(dilation=2), "dilation"), (dict(dilation=[1, 1]), "dilation"), (dict(weights=[1.0, 0.5]), "weights")):
        with pytest.raises(ValueError, match=match):
            disparity_loss.forward(_Loss(**kw), x, lab)
    # the reference's own call turns weights / dilation into [1.0] / [1]: still the shipped settings (then refused for the CPU tensors)
    with pytest.raises(RuntimeError, match="CUDA"):
        disparity_loss.check_criterion(_Crit(weights=[1.0], dilation=[1]))
        disparity_loss.disparity_loss(x, lab)


def test_install_disparity_loss_into_reference():
    import refload
    if not refload.available():
        pytest.skip("reference package not available")
    refload.load_reference()
    from visualDet3D.networks.heads import detection_3d_head, losses
    from visualdet3d_b200 import plugin
    orig, anchor = losses.DisparityLoss.forward, detection_3d_head.AnchorBasedDetection3DHead.loss
    try:
        fn = plugin.install_disparity_loss_into_reference()
        assert fn is disparity_loss.forward and losses.DisparityLoss.forward is disparity_loss.forward
        assert detection_3d_head.AnchorBasedDetection3DHead.loss is anchor
        with pytest.raises(RuntimeError, match="CUDA"):                      # the reference module now runs the native loss
            losses.DisparityLoss(96)(torch.zeros(1, 96, 2, 2), torch.ones(1, 2, 2))
    finally:
        losses.DisparityLoss.forward = orig
