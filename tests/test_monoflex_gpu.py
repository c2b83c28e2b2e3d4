"""-m gpu: MonoFlex (DLA-34 + DCNv2 up-sampling + CenterNet heads/decode) against the reference fixtures and the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_fixture, subsample_like
import torch_port as tp
from detector_harness import match_dets, run_with_stages

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mf():
    from visualdet3d_b200.detectors import build_synthetic_monoflex
    det, sd, cfg = build_synthetic_monoflex(seed=0)
    return det.cuda().eval(), sd, cfg


@pytest.mark.parametrize("tag", ["monoflex_96x320", "monoflex_192x640", "monoflex_384x1280"])     # the last one = BASELINE configs[3] shape
def test_against_reference_fixture(mf, tag):
    from visualdet3d_b200 import synth
    det, sd, cfg = mf
    fx = load_fixture(tag)
    H, W, B, seed = [int(v) for v in fx["meta"]]
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
    res, st = run_with_stages(det, img, P2)
    rep = {"features": float(np.abs(subsample_like(st["features"], fx["features"]) - fx["features"]["samples"]).max())}
    off = det._plan["offsets"]
    for n, k in cfg["head"]["layer_cfg"]["head_dict"].items():
        got = st["heads"][:, off[n]:off[n] + k]
        rep[n] = float(np.abs(subsample_like(got, fx["head_" + n]) - fx["head_" + n]["samples"]).max())
    print(tag, "stage max|diff| vs reference:", rep)
    assert all(v < 1e-3 for v in rep.values()), rep
    ref = tp.monoflex_forward(sd, img, P2, cfg)
    for b in range(B):
        k = len(res[b][0])
        assert k == len(fx[f"scores_{b}"])
        match_dets(res[b], ref[b], det._last_decoder.anchor[b, :k])
        # ... and against the reference's own outputs (same rows: the oracle equals the fixture row for row, test_oracle_golden.py)
        if torch.equal(det._last_decoder.anchor[b, :k].cpu().long(), ref[b][3]):
            np.testing.assert_allclose(res[b][0].cpu().numpy(), fx[f"scores_{b}"], atol=1e-3, rtol=0)
            np.testing.assert_allclose(res[b][1].cpu().numpy(), fx[f"bboxes_{b}"], atol=1e-3, rtol=1e-5)
            np.testing.assert_array_equal(res[b][2].cpu().numpy().reshape(-1), fx[f"cls_{b}"].reshape(-1))


def test_lo_companions_are_fresh_everywhere(mf, monkeypatch):
    """VD3D_CHECK_LO: in front of every tensor-core conv of the DLA / DLAUp / head plan the fp16 (hi, lo) planes must equal the split of the fp32 tensor:
    the plan skips the split pass for views whose producer wrote the planes itself (`Act.lo_fresh`), and splits only the copied children of a Root concat."""
    from visualdet3d_b200 import synth, engine
    det = mf[0]
    monkeypatch.setattr(engine, "CHECK_LO", True)
    img, P2 = synth.synth_mono_inputs(2, 96, 320, seed=6)
    with torch.no_grad():
        det.forward_batch(img.cuda(), P2.cuda())


def test_batch8_384x1280_all_images_vs_oracle(mf):
    """BASELINE configs[3] shape (DLA-34 + DCNv2, batch 8, 384x1280): determinism, batch invariance, and EVERY image of the
    batch against the oracle."""
    from visualdet3d_b200 import synth
    det, sd, cfg = mf
    img, P2 = synth.synth_mono_inputs(8, 384, 1280, seed=9)
    ic, pc = img.cuda(), P2.cuda()
    with torch.no_grad():
        r1 = det.forward_batch(ic, pc)
        idx = [det._last_decoder.anchor[b, :len(r1[b][0])].clone() for b in range(8)]
        r2 = det.forward_batch(ic, pc)
        single = det([ic[2:3], pc[2:3]])
    assert all(torch.equal(x, y) for a, b in zip(r1, r2) for x, y in zip(a, b))
    assert all(torch.equal(x, y) for x, y in zip(r1[2], single))
    ref = tp.monoflex_forward(sd, img, P2, cfg)
    for b in range(8):
        match_dets(r1[b], ref[b], idx[b])
    print("MonoFlex 8 x 384x1280: detections per image", [len(r[0]) for r in r1])


def heads_to_act(det, outs):
    """oracle head maps {name: [B, n, H, W]} -> the NHWC tensor layout `decode_maps` reads (channel offsets of the plan)."""
    from visualdet3d_b200 import engine as E
    pl = det.prepare()
    any_map = next(iter(outs.values()))
    B, _, h, w = any_map.shape
    t = torch.zeros(B, h, w, pl["out_channels"])
    for n, v in outs.items():
        t[..., pl["offsets"][n]:pl["offsets"][n] + v.shape[1]] = v.permute(0, 2, 3, 1)
    return E.Act(t.cuda().contiguous())


@pytest.mark.parametrize("kind,H,W,B", [("KM3D", 192, 640, 2), ("KM3D", 384, 1280, 1), ("MonoFlex", 384, 1280, 1)])
def test_centernet_decode_on_oracle_maps(kind, H, W, B):
    """The decode kernels in isolation, fed with the ORACLE's head maps (no network error in front of them): peak sets and order
    bit-exact, every output column within 1e-3 -- including the KM3D positions (float64 3x3 normal equations on both sides)."""
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_monoflex
    det, sd, cfg = build_synthetic_monoflex(seed=0, name=kind)
    det = det.cuda().eval()
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=3)
    st = {}
    ref = (tp.km3d_forward if kind == "KM3D" else tp.monoflex_forward)(sd, img, P2, cfg, st)
    with torch.no_grad():
        dec = det.decode_maps(heads_to_act(det, st["heads"]), P2.cuda(), H, W)
    out = dec.results()
    worst = np.zeros(11)
    for b in range(B):
        rs, rb, rc, rflat = ref[b]
        k = len(rs)
        assert len(out[b][0]) == k and k > 3
        assert torch.equal(dec.anchor[b, :k].cpu().long(), rflat), "peak indices / order differ"
        assert torch.equal(out[b][2].cpu().view(-1), rc.view(-1))
        np.testing.assert_allclose(out[b][0].cpu().numpy(), rs.numpy(), atol=1e-6, rtol=0)
        worst = np.maximum(worst, (out[b][1].cpu() - rb).abs().max(0)[0].numpy())
    print(kind, f"{H}x{W} decode on oracle maps: max |diff| per column", np.array2string(worst, precision=2))
    assert float(worst.max()) < 1e-3, worst


@pytest.mark.parametrize("tag", ["km3d_96x320", "km3d_192x640", "km3d_384x1280"])     # the last one = BASELINE configs[3] shape
def test_km3d_against_reference_fixture_and_oracle(tag):
    """KM3D: same network family, keypoint-refined least-squares decode (km3d_head.py:155-314, rtm3d_utils.py:314-455)."""
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_monoflex
    det, sd, cfg = build_synthetic_monoflex(seed=0, name="KM3D")
    det = det.cuda().eval()
    fx = load_fixture(tag)
    H, W, B, seed = [int(v) for v in fx["meta"]]
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
    res, st = run_with_stages(det, img, P2)
    off = det._plan["offsets"]
    rep = {}
    for n, k in cfg["head"]["layer_cfg"]["head_dict"].items():
        got = st["heads"][:, off[n]:off[n] + k]
        rep[n] = float(np.abs(subsample_like(got, fx["head_" + n]) - fx["head_" + n]["samples"]).max())
    print(tag, "head max|diff| vs reference:", rep)
    assert all(v < 1e-3 for v in rep.values()), rep
    ref = tp.km3d_forward(sd, img, P2, cfg)
    # The reference is not deterministic here: gen_position adds randn * 1e-8 to the float64 normal matrix before inverting it
    # (rtm3d_utils.py:447).  tests/golden/km3d_spread.npz holds the [min, max] envelope of every output entry over 8 torch seeds of the
    # UNMODIFIED reference (make_golden_km3d_spread.py): at 384x1280 its own spread reaches 2.3e-3 in z (22 of 100 rows above 1e-3).
    # Bar: every column within 1e-3 of the oracle, except the three position-derived columns (cx, cy, z), which must lie within
    # 1e-3 + the reference's own spread of that entry from the reference's envelope.
    env = np.load(os.path.join(GOLDEN, "km3d_spread.npz"))
    for b in range(B):
        k = len(res[b][0])
        assert k == len(fx[f"scores_{b}"])
        gi = det._last_decoder.anchor[b, :k].cpu().long()
        rs, rb, rc, rflat = ref[b]
        assert torch.equal(torch.sort(gi)[0], torch.sort(rflat)[0]), "kept peak sets differ"
        pos = {int(a): i for i, a in enumerate(rflat.tolist())}
        perm = torch.tensor([pos[int(a)] for a in gi.tolist()])
        s, bx, ci = [t.cpu() for t in res[b]]
        for i in (perm != torch.arange(k)).nonzero()[:, 0].tolist():
            assert abs(float(rs[perm[i]]) - float(rs[i])) < 1e-5, "order differs between rows that are not score-tied"
        assert torch.equal(ci.view(-1), rc[perm].view(-1))
        assert float((s - rs[perm]).abs().max()) < 1e-3
        d = (bx - rb[perm]).abs().numpy()
        lo, hi = env[f"{H}x{W}_{b}/min"][perm.numpy()], env[f"{H}x{W}_{b}/max"][perm.numpy()]
        out_of_env = np.maximum(lo - bx.numpy(), bx.numpy() - hi).clip(min=0)
        spread = (hi.astype(np.float64) - lo).astype(np.float32)
        print(tag, b, "max |diff| vs oracle per column", np.array2string(d.max(0), precision=2),
              "| distance to the reference envelope", np.array2string(out_of_env.max(0), precision=2),
              "| reference spread", np.array2string(spread.max(0), precision=2))
        other = [0, 1, 2, 3, 7, 8, 9, 10]
        assert float(d[:, other].max()) < 1e-3, d[:, other].max(0)
        assert bool((out_of_env[:, 4:7] <= 1e-3 + spread[:, 4:7]).all()), (out_of_env[:, 4:7] - spread[:, 4:7]).max(0)
