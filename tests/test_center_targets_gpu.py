"""KM3D / MonoFlex target kernels (`vd3d_center_targets`, visualdet3d_b200/center_targets.py:DeferredTargetBatch.to_device) against their
host form on the fixture cases of tests/golden/center_targets.npz: bit for bit, batched with mixed object counts and at B = 32, the same
bits on a second run, two launches per batch; the device dict gives km3d_head_loss / monoflex_head_loss the loss the reference's
targets give; and the reference's datasets, collate_fn and train_rtm3d with the targets install, alone and with the augmentation
install, hand the module the reference's inputs."""
import numpy as np
import pytest
import torch

from visualdet3d_b200 import _lib
from visualdet3d_b200 import center_targets as ct
from test_center_targets_cpu import CASES, FX, deferred, targets

pytestmark = pytest.mark.gpu


def _by_mode(mode):
    return [k for k in CASES if int(FX[k]["mode"]) == mode and not int(FX[k]["raises"])]


def _run(ts):
    _lib.launch_count_reset()
    got = ct.DeferredTargetBatch(ts).pin_memory().to_device("cuda")
    torch.cuda.synchronize()
    assert _lib.launch_count() == 2
    return got


def _same(got, ts):
    for i, t in enumerate(ts):
        want = ct.build_targets_host(t)
        assert list(got) == list(want)
        for key, w in want.items():
            g = got[key][i].cpu().numpy()
            assert g.dtype == w.dtype and g.shape == w.shape, key
            assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), (key, i)


@pytest.mark.parametrize("case", CASES)
def test_kernel_matches_host_form_per_case(case):
    if int(FX[case]["raises"]):
        pytest.skip("the reference raises: nothing is launched")
    ts = [deferred(FX[case])]
    _same(_run(ts), ts)


@pytest.mark.parametrize("mode", [ct.MODE_KM3D, ct.MODE_MONOFLEX])
def test_kernel_matches_host_form_batched(mode):
    """Mixed object counts in one batch (0 ... 32), then B = 32; a second run gives the same bits."""
    ts = [deferred(FX[k]) for k in _by_mode(mode) if tuple(FX[k]["hw"]) == (384, 1280)]
    assert len({int(t.record.view(np.int32)[-6]) for t in ts}) >= 4
    got = _run(ts)
    _same(got, ts)
    big = (ts * 32)[:32]
    got = _run(big)
    _same(got, big)
    again = _run(big)
    for key in got:
        assert torch.equal(got[key], again[key]), key


def _maps(mode, B, C, h, w, seed):
    from visualdet3d_b200 import km3d_loss, monoflex_loss
    g = torch.Generator(device="cuda").manual_seed(seed)
    maps = (monoflex_loss if mode else km3d_loss).MAPS
    return {name: (torch.randn(B, c or C, h, w, generator=g, device="cuda") * 0.5).contiguous() for name, c in maps}


@pytest.mark.parametrize("mode", [ct.MODE_KM3D, ct.MODE_MONOFLEX])
def test_loss_on_device_targets_matches_reference_targets(mode):
    from visualdet3d_b200.km3d_loss import km3d_head_loss
    from visualdet3d_b200.monoflex_loss import monoflex_head_loss
    keys = [k for k in _by_mode(mode) if tuple(FX[k]["hw"]) == (384, 1280) and FX[k]["objs"].shape[0] > 0]
    ts = [deferred(FX[k]) for k in keys]
    dev = _run(ts)
    ref = {key: torch.from_numpy(np.stack([targets(FX[k])[key] for k in keys])).cuda() for key in dev}
    P2 = torch.from_numpy(np.stack([FX[k]["P2"] for k in keys])).float().cuda()
    out = _maps(mode, len(keys), 3, 96, 320, seed=mode)
    if mode == ct.MODE_KM3D:
        a, _ = km3d_head_loss(out, dev, P2, epoch=5)
        b, _ = km3d_head_loss(out, ref, P2, epoch=5)
    else:
        a, _ = monoflex_head_loss(out, dev, P2)
        b, _ = monoflex_head_loss(out, ref, P2)
    a, b = float(a), float(b)
    print(f"mode {mode}: loss on device targets {a:.9g}, on the reference's {b:.9g}")
    assert np.isfinite(a) and abs(a - b) <= 1e-6 * abs(b)


def test_plugin_matches_the_reference_training_input(tmp_path):
    """KittiRTM3DDataset and KittiMonoFlexDataset + collate_fn + train_rtm3d, as shipped, with the targets install, and with both installs,
    from the same seed: the module gets the same keys, dtypes and shapes, the targets within the host-form rules, and images within the
    augmentation's bound."""
    from loss_harness import run_seam_worker
    out = run_seam_worker("center_targets_plugin.py", str(tmp_path))
    assert set(out) == {f"{ds}_{arm}" for ds in ("km3d", "monoflex") for arm in ("targets", "both")}
    for arm, r in out.items():
        assert r["keys_equal"] and r["dtypes_shapes_equal"] and r["exact_equal"] and r["float_close"], (arm, r)
        assert r["targets_on_gpu"] and r["rng_equal"] and r["P2_equal"], (arm, r)
        assert r["image_max_diff"] <= (5e-5 if arm.endswith("both") else 0.0), (arm, r)
