"""CPU checks of the RetinaNet 2-D detector: state_dict contract, anchors, config refusals, opt-in install into the reference."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_fixture, subsample_like

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import refload  # noqa: E402


def build(**kw):
    from visualdet3d_b200 import synth
    from visualdet3d_b200.plugin import DETECTOR_DICT
    import visualdet3d_b200.detectors  # noqa: F401
    cfg = synth.retinanet_cfg(**kw)
    return DETECTOR_DICT["RetinaNet"](cfg), cfg


def test_state_dict_keys_and_shapes_match_reference():
    det, _ = build()
    ref = json.load(open(os.path.join(GOLDEN, "retinanet_keys.json")))
    ours = {k: list(v.shape) for k, v in det.state_dict().items()}
    assert list(ours) == list(ref)
    assert ours == ref


@pytest.mark.parametrize("tag", ["retinanet_96x320", "retinanet_288x1280", "retinanet_64x128_nopre"])
def test_anchors_bit_exact(tag):
    from visualdet3d_b200.anchors import grid_anchors
    det, _ = build()
    fx = load_fixture(tag)
    H, W = int(fx["meta"][0]), int(fx["meta"][1])
    a = det.anchors_cfg
    got = torch.tensor(grid_anchors((H, W), a["pyramid_levels"], a["strides"], a["sizes"], a["ratios"], a["scales"]).astype(np.float32))
    np.testing.assert_array_equal(subsample_like(got, fx["anchors"]), fx["anchors"]["samples"])
    if "anchors_full" in fx:
        np.testing.assert_array_equal(got.numpy(), fx["anchors_full"])


def test_config_refusals():
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors.retinanet import RetinaNet
    cfg = synth.retinanet_cfg()
    cfg.neck.num_outs = 2
    with pytest.raises(ValueError, match="num_outs"):
        RetinaNet(cfg)
    cfg = synth.retinanet_cfg(nms_pre=5000)
    with pytest.raises(ValueError, match="capacity"):
        RetinaNet(cfg)
    cfg = synth.retinanet_cfg()
    cfg.backbone.pretrained = True
    with pytest.raises(RuntimeError, match="pretrained"):
        RetinaNet(cfg)
    cfg = synth.retinanet_cfg()
    cfg.head.test_cfg.cls_agnositc = False
    with pytest.raises(ValueError, match="class-aware"):
        RetinaNet(cfg)
    cfg = synth.retinanet_cfg()
    cfg.neck.in_channels = [256, 512, 1024]
    with pytest.raises(ValueError, match="channels"):
        RetinaNet(cfg)
    det, _ = build()
    with pytest.raises(NotImplementedError):
        det([torch.zeros(1, 3, 64, 64), None, None])
    with pytest.raises(RuntimeError, match="CPU"):                  # no CPU path: fails loudly (Vd3dError)
        det([torch.zeros(1, 3, 64, 64), None])


_INSTALL_WORKER = r"""
import json, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/oracle")
import refload
refload.load_reference()
from visualDet3D.networks.utils import registry as ref
from visualdet3d_b200 import plugin
import visualdet3d_b200.detectors  # noqa
plugin.install_into_reference()
after_all = ref.DETECTOR_DICT["RetinaNet"].__module__
plugin.install_retinanet_into_reference()
print("JSON " + json.dumps([after_all, ref.DETECTOR_DICT["RetinaNet"].__module__]))
"""


@pytest.mark.skipif(not refload.available(), reason="no reference package")
def test_install_retinanet_is_opt_in():
    r = subprocess.run([sys.executable, "-c", _INSTALL_WORKER, ROOT], capture_output=True, text=True, timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("JSON ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:] + r.stderr[-2000:]
    after_all, after_opt_in = json.loads(lines[-1][5:])
    assert after_all.startswith("visualDet3D.")                  # install_into_reference() leaves the reference's RetinaNet
    assert after_opt_in == "visualdet3d_b200.detectors.retinanet"
