"""The test-time input pipeline on the device, bit for bit against the SHA-256 digests of tests/golden/make_golden_preprocess_digests.py
(recorded from the host form): `preprocess_batch` with every frame of one geometry in one launch, and the network-input buffers that
`StreamedInference.submit_frames` fills for a stereo detector (both cameras; a frame smaller than the staging frame is stored top-left, so
its rows are the staging frame's pitch apart).  Input the kernel's 2x stage or its 3-channel layout cannot take is refused before any
launch."""
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from visualdet3d_b200 import _lib
from visualdet3d_b200 import preprocess as pp

sys.path.insert(0, GOLDEN)
from make_golden_preprocess_digests import OUT, cases, digest  # noqa: E402

pytestmark = pytest.mark.gpu


def test_preprocess_batch_matches_digests():
    fx = np.load(OUT)
    groups = {}
    for c in cases():
        groups.setdefault((c["id"].split("/")[0], c["crop_top"], c["size"]), []).append(c)
    n = 0
    for (_, crop, size), cs in groups.items():
        got = pp.preprocess_batch([c["frame"] for c in cs], crop, size, cs[0]["mean"], cs[0]["std"]).cpu().numpy()
        for c, g in zip(cs, got):
            assert digest(g) == str(fx[c["id"]]), c["id"]
            n += 1
    assert n == len(fx.files)


# (left, right) frames of each sample, one batch per geometry: the fixture's 370 x 1224 pair shares a batch with a 375 x 1242 pair
PIPELINE_BATCHES = [[("fixture/c0_l", "fixture/c0_r"), ("fixture/c1_l", "fixture/c1_r")], [("fixture/c2_l", "fixture/c2_r")],
                    [("fixture/c3_l", "fixture/c3_r")], [("bench/crop2_384x1280_s0", "bench/crop2_384x1280_s1")],
                    [("bench/crop96_288x1280_s0", "bench/crop96_288x1280_s1")]]


def test_submit_frames_fills_the_network_inputs_of_the_digests():
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    from visualdet3d_b200.pipeline import StreamedInference
    fx = np.load(OUT)
    by_id = {c["id"]: c for c in cases()}
    det = build_synthetic_stereo3d(seed=0)[0].cuda().eval()
    for pairs in PIPELINE_BATCHES:
        first = by_id[pairs[0][0]]
        hw = [by_id[left]["frame"].shape[:2] for left, _ in pairs]
        B, (H, W), Hf, Wf = len(pairs), first["size"], max(h for h, _ in hw), max(w for _, w in hw)
        staged = [torch.zeros(B, Hf, Wf, 3, dtype=torch.uint8) for _ in range(2)]
        for b, pair in enumerate(pairs):
            for cam, cid in enumerate(pair):
                f = by_id[cid]["frame"]
                staged[cam][b, :f.shape[0], :f.shape[1]] = torch.from_numpy(f)
        pipe = StreamedInference(det, B, H, W, kmax=64, frame_hw=(Hf, Wf), crop_top=first["crop_top"])
        P2 = synth.synth_stereo_inputs(B, H, W, seed=3)[2]
        t = pipe.submit_frames(*[s.pin_memory() for s in staged], P2.pin_memory(), sizes=hw)
        torch.cuda.synchronize()
        for cam in range(2):
            got = pipe.bufs[t % pipe.depth][cam].cpu().numpy()
            for b, pair in enumerate(pairs):
                assert digest(got[b]) == str(fx[pair[cam]]), pair[cam]


def test_refused_before_any_launch():
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_mono3d
    from visualdet3d_b200.pipeline import StreamedInference
    det = build_synthetic_mono3d("Yolo3D", seed=0)[0].cuda().eval()
    pipe = StreamedInference(det, 1, 96, 320, kmax=64, frame_hw=(300, 700), crop_top=0)          # a 3.125x source step
    torch.cuda.synchronize()
    _lib.launch_count_reset()
    with pytest.raises(_lib.Vd3dError, match="shrinks"):
        pp.preprocess_batch([np.zeros((40, 20, 3), np.uint8)], 0, (8, 16))
    with pytest.raises(_lib.Vd3dError, match="bad arguments"):
        pp.preprocess_batch([np.zeros((10, 20, 4), np.uint8)], 2, (8, 16))
    with pytest.raises(_lib.Vd3dError, match="shrinks"):
        pipe.submit_frames(torch.zeros(1, 300, 700, 3, dtype=torch.uint8).pin_memory(), synth.synth_mono_inputs(1, 96, 320)[1].pin_memory())
    torch.cuda.synchronize()
    assert _lib.launch_count() == 0
