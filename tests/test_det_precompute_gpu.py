"""The anchor-prior kernels and the det_precompute CLI on the GPU: the device accumulation against the host entry on every constructed
case (bit for bit, twice), input checks, and the CLI's files against the unmodified reference script's (tests/golden/det_precompute.npz;
the reference script itself, run on the same GPU, when oracle/_ref/scripts was built)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import det_precompute_cases as dc

pytestmark = pytest.mark.gpu
CASES = {c["id"]: c for c in dc.kernel_cases()}


@pytest.fixture(scope="module")
def fx():
    z = np.load(os.path.join(GOLDEN, "det_precompute.npz"))
    return {k: z[k] for k in z.files}


def device_state(c):
    import torch
    from visualdet3d_b200 import anchor_prior as ap
    st = ap.PriorState(c["T"], c["n_bins"], "cuda")
    order, start = ap.bin_order(c["bins"], c["n_bins"])
    ap.accumulate(st, torch.from_numpy(c["anchors"]).cuda(), torch.from_numpy(order).cuda(), start, c["offsets"],
                  torch.from_numpy(c["boxes"]).cuda(), torch.from_numpy(c["gt3"]).cuda(), c["thr"])
    return st.numpy()


@pytest.mark.parametrize("cid", sorted(CASES))
def test_device_equals_host_and_golden(cid, fx):
    from visualdet3d_b200 import anchor_prior as ap
    c = CASES[cid]
    host = ap.PriorState(c["T"], c["n_bins"])
    order, start = ap.bin_order(c["bins"], c["n_bins"])
    ap.accumulate_host(host, c["anchors"], order, start, c["offsets"], c["boxes"], c["gt3"], c["thr"])
    a, b = device_state(c), device_state(c)
    for k in ("examine", "sums", "squared", "usable"):
        np.testing.assert_array_equal(a[k], host.numpy()[k], err_msg=f"{cid} {k}")
        np.testing.assert_array_equal(a[k], fx[f"case/{cid}/{k}"], err_msg=f"{cid} {k}")
        assert a[k].tobytes() == b[k].tobytes()


def test_batches_carry_the_state():
    """Two launches of half the frames each give the bits of one launch over all of them."""
    import torch
    from visualdet3d_b200 import anchor_prior as ap
    c = CASES["many_frames_f32"]
    order, start = ap.bin_order(c["bins"], c["n_bins"])
    whole = device_state(c)
    st = ap.PriorState(c["T"], c["n_bins"], "cuda")
    half = c["B"] // 2 * c["T"]
    for s0, s1 in ((0, half), (half, c["B"] * c["T"])):
        off = c["offsets"][s0:s1 + 1]
        ap.accumulate(st, torch.from_numpy(c["anchors"]).cuda(), torch.from_numpy(order).cuda(), start, off - off[0],
                      torch.from_numpy(c["boxes"][off[0]:off[-1]]).cuda(), torch.from_numpy(c["gt3"][off[0]:off[-1]]).cuda(), c["thr"])
    for k, v in st.numpy().items():
        assert v.tobytes() == whole[k].tobytes(), k


def test_bad_inputs_raise():
    import torch
    from visualdet3d_b200 import anchor_prior as ap
    c = CASES["tied_gts"]
    order, start = ap.bin_order(c["bins"], c["n_bins"])
    st = ap.PriorState(1, 1, "cuda")
    a, o = torch.from_numpy(c["anchors"]).cuda(), torch.from_numpy(order).cuda()
    bx, g = torch.from_numpy(c["boxes"]).cuda(), torch.from_numpy(c["gt3"]).cuda()
    ap.accumulate(st, a, o, start, c["offsets"], bx, g, 0.5)
    with pytest.raises(ValueError):
        ap.accumulate(st, a.cpu(), o, start, c["offsets"], bx, g, 0.5)
    with pytest.raises(TypeError):
        ap.accumulate(st, a, o, start, c["offsets"], bx.half(), g, 0.5)
    with pytest.raises(TypeError):
        ap.accumulate(st, a, o, start, c["offsets"], bx, g.float(), 0.5)
    with pytest.raises(ValueError):
        ap.accumulate(st, a, o, start, np.array([0, 3]), bx, g, 0.5)          # offsets end past the boxes
    with pytest.raises(ValueError):
        ap.accumulate(st, a, o, start, np.array([0, 2, 1]), bx, g, 0.5)       # not B * T + 1 values
    with pytest.raises(ValueError):
        ap.accumulate(st, a, o, np.array([0, 2]), c["offsets"], bx, g, 0.5)   # bins past N
    with pytest.raises(ValueError):
        ap.accumulate(st, a, o, start, torch.from_numpy(c["offsets"]).cuda(), bx, g, 0.5)
    with pytest.raises(ValueError):
        ap.accumulate(st, a, o, start, c["offsets"], bx, g[:1], 0.5)


CLI = """import os, runpy, sys
ROOT = sys.argv[1]
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import refload
from visualdet3d_b200.ops import dcn, iou3d
refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
sys.argv = ["det_precompute"] + sys.argv[2:]
runpy.run_module("visualdet3d_b200.det_precompute", run_name="__main__")
"""

REF = """import os, sys
ROOT, cfgp = sys.argv[1], sys.argv[2]
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
import refload
from visualdet3d_b200.ops import dcn, iou3d
refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
import make_golden_det_precompute as mg
mod, _ = mg.reference_scripts(os.path.join(ROOT, "oracle", "_ref", "scripts"), cpu=False)
from visualDet3D.utils.utils import cfg_from_file
cfg = cfg_from_file(cfgp)
tr, _ = mod.process_train_val_file(cfg)
mod.read_one_split(cfg, tr, cfg.path.data_path, {"calib": True, "image": True, "label": True, "velodyne": False}, 'training', 100)
"""


FLAT = """import os, sys
ROOT, tmp, out = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
import numpy as np
import refload
from visualdet3d_b200.ops import dcn, iou3d
refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
import make_golden_det_precompute as mg
flat = {}
for a in sys.argv[4:]:
    prefix, path = a.split("=", 1)
    mg.flatten_pickle(path, tmp, prefix, flat)
np.savez(out, **{k.replace("/", "|"): v for k, v in flat.items()})
"""


def _run(script, *args, cwd):
    r = subprocess.run([sys.executable, "-c", script, ROOT, *args], capture_output=True, text=True, cwd=cwd, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


def test_cli_writes_the_reference_files(fx):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import refload
    with tempfile.TemporaryDirectory() as tmp:
        raw, split = dc.write_tree(tmp)
        for name in dc.CONFIGS:
            cfgp = dc.write_config(name, tmp, raw, split)
            _run(CLI, f"--config={cfgp}", "--split=train", cwd=tmp)
            pre = os.path.join(tmp, "pre", name)
            for sp in ("training", "validation"):
                d = os.path.join(pre, sp)
                npys = sorted(f[:-4] for f in os.listdir(d) if f.endswith(".npy"))
                assert npys == sorted(k[len(f"{name}/{sp}/"):] for k in fx if k.startswith(f"{name}/{sp}/anchor_"))
                for f in npys:
                    np.testing.assert_array_equal(np.load(os.path.join(d, f + ".npy")), fx[f"{name}/{sp}/{f}"], err_msg=f"{name} {f}")
                npz = os.path.join(tmp, "flat.npz")
                _run(FLAT, tmp, npz, f"{name}/{sp}/pkl/=" + os.path.join(d, "imdb.pkl"), cwd=tmp)
                z = np.load(npz)
                out = {k.replace("|", "/"): z[k] for k in z.files}
                assert sorted(out) == sorted(k for k in fx if k.startswith(f"{name}/{sp}/pkl/"))
                for k, v in out.items():
                    np.testing.assert_array_equal(v, fx[k], err_msg=k)
        # the native Stereo3D's prior loader takes the CLI's files: [T, 16 scales, 3 ratios, 6]
        from visualdet3d_b200.anchors import AnchorTable, load_priors
        m, s = load_priors(os.path.join(tmp, "pre", "stereo3d"), ["Car", "Pedestrian"], 16, 3)
        cfg = dict(pyramid_levels=[4], strides=[16], sizes=[24], ratios=np.array([0.5, 1, 2.0]),
                   scales=np.array([2 ** (i / 4.0) for i in range(16)]))
        t = AnchorTable((288, 1280), cfg, m, s, "cuda")
        assert t.N == 69120 and t.mean_std.shape == (69120, 2, 6, 2)
        if refload.available() and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "scripts")):
            for name in ("stereo3d", "stereo3d_f64"):          # the unmodified script on this GPU: a second oracle
                cfgp = dc.write_config(name, os.path.join(tmp, "refrun"), raw, split)
                _run(REF, cfgp, cwd=tmp)
                d = os.path.join(tmp, "refrun", "pre", name, "training")
                for f in sorted(os.listdir(d)):
                    if f.endswith(".npy"):
                        np.testing.assert_array_equal(np.load(os.path.join(tmp, "pre", name, "training", f)), np.load(os.path.join(d, f)),
                                                      err_msg=f"{name} {f} vs the reference on the GPU")


def test_accumulator_follows_each_segments_dtype_on_the_device():
    """The device accumulator launches each segment in its own IoU dtype, frames and classes mixing them, with the host entry's bits."""
    from visualdet3d_b200.anchor_prior import AnchorPriorAccumulator
    states = []
    for device in (None, "cuda"):
        acc = AnchorPriorAccumulator(dc.FLIP_CFG, (16, 16), ["Car", "Pedestrian"], 0.6, device)
        acc.add(dc.dtype_frames())
        states.append(acc.state.numpy())
    assert states[1]["examine"][:, 0].tolist() == [2, 1] and states[1]["usable"].tolist() == [2, 1]
    for k, v in states[0].items():
        assert v.tobytes() == states[1][k].tobytes(), k


def test_workspace_budget_is_enforced():
    import torch
    from visualdet3d_b200 import anchor_prior as ap
    N, T = 69120, 2
    B = ap.max_frames_per_launch(N, T) + 1
    st = ap.PriorState(T, 48, "cuda")
    a = torch.zeros((N, 4), device="cuda")
    o = torch.arange(N, dtype=torch.int32, device="cuda")
    start = np.linspace(0, N, 49).astype(np.int32)
    with pytest.raises(ValueError, match="workspace"):
        ap.accumulate(st, a, o, start, np.zeros(B * T + 1, np.int32), torch.zeros((0, 4), device="cuda"),
                      torch.zeros((0, 3), dtype=torch.float64, device="cuda"), 0.5)
