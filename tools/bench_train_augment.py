"""Time the training-time augmentation: the reference's host chain (cv2 / numpy `Compose` of the shipped train_augmentation list) against
the GPU form (visualdet3d_b200/train_augment.py: host draws + `augment_batch`, one kernel per batch), on two configurations:
  stereo:   batch 8 stereo pairs (16 images), 375x1242 -> 288x1280, chain 1 (Stereo3D_example: photometric program, CropTop, Resize);
  monoflex: batch 8 images, 375x1242 -> 384x1280, chain 2 (Monoflex_example: warp on uint8, Shuffle'd photometric program).

Reports, per configuration:
  * the reference chain's host time per sample on one core, and samples/s with `--workers` processes (the shipped num_workers = 4);
  * the host part of the GPU form per sample (the same random draws, calibration and label updates; no image work);
  * the kernel time per batch from CUDA events over `--launches` back-to-back launches after warm-up, with its algorithmic bytes (the uint8
    frame rows the geometry reads plus the float32 output) as GB/s and as a share of 3.35 TB/s;
  * augment_batch per batch (pinned staging copy, upload, descriptors, kernel; host clock ending in a device synchronise);
and one train_stereo_detection step of the reference Stereo3D with the native losses, fed by the reference dataset + collate_fn with and
without `plugin.install_train_augmentation_into_reference()` (train_step_arm).
Prints one JSON line with the card's name, power limit and max SM clock; writes nothing.

    python tools/bench_train_augment.py [--samples 32] [--workers 4] [--launches 200] [--steps 20] [--warmup 5]
The reference arm needs the reference package and cv2; without them only the GPU arm runs."""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time
import types
from copy import deepcopy

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402
import train_augment_cases as cases  # noqa: E402
from bench_common import card  # noqa: E402
from visualdet3d_b200 import _lib  # noqa: E402
from visualdet3d_b200 import train_augment as ta  # noqa: E402

HBM_BYTES_PER_S = 3.35e12        # H100 SXM5 80 GB HBM3
H, W, BATCH = 375, 1242, 8
CONFIGS = {"stereo": "stereo3d", "monoflex": "monoflex"}


def _inputs(name, i, make=types.SimpleNamespace):
    return cases.frame(i, H, W), cases.frame(i + 1, H, W), cases.P2.copy(), cases.P3.copy(), cases.labels(i, H, W, make)


def _call(aug, stereo, x):
    left, right, p2, p3, lab = x
    return aug(left, right, p2, p3, lab) if stereo else aug(left, p2=p2, labels=lab)


def _ref_worker(args):
    """One process on one cv2 thread: the reference chain over `n` samples, seconds spent in the transform calls only."""
    name, n, seed = args
    import cv2
    cv2.setNumThreads(1)
    import refload
    refload.load_reference()
    from visualDet3D.data.pipeline import build_augmentator
    from visualDet3D.data.kitti.kittidata import KittiObj
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_train_augment import edict
    aug_list, stereo = cases.LISTS[name]
    compose = build_augmentator(edict(aug_list))
    xs = [_inputs(name, seed + i, KittiObj) for i in range(n)]
    np.random.seed(seed)
    _call(compose, stereo, deepcopy(xs[0]))                            # warm-up
    t0 = time.perf_counter()
    for x in xs:
        _call(compose, stereo, x)
    return t0, time.perf_counter()


def reference_arm(name, samples, workers):
    try:
        import cv2  # noqa: F401
        import refload
        if not refload.available():
            return {"reference": "not measured (no reference package)"}
    except ImportError:
        return {"reference": "not measured (no cv2)"}
    ctx = mp.get_context("spawn")
    with ctx.Pool(1) as pool:
        t0, t1 = pool.map(_ref_worker, [(name, samples, 0)])[0]
        one = t1 - t0
    with ctx.Pool(workers) as pool:
        # each worker times only its transform loop; the span from the first start to the last end is the parallel wall time
        spans = pool.map(_ref_worker, [(name, samples, 100 * k) for k in range(workers)], chunksize=1)
        wall = max(e for _, e in spans) - min(s for s, _ in spans)
    return {"reference_ms_per_sample_1core": round(one * 1e3 / samples, 2),
            f"reference_samples_per_s_{workers}workers": round(workers * samples / wall, 1)}


def gpu_arm(name, samples, launches):
    aug_list, stereo = cases.LISTS[name]
    aug = ta.TrainAugmentation(aug_list)
    xs = [_inputs(name, i) for i in range(samples)]
    np.random.seed(0)
    t0 = time.perf_counter()
    outs = [_call(aug, stereo, x) for x in xs]
    host_ms = (time.perf_counter() - t0) * 1e3 / samples
    batches = []
    for b in range(0, samples - BATCH + 1, BATCH):
        group = outs[b:b + BATCH]
        batches.append([o[0] for o in group] + ([o[1] for o in group] if stereo else []))
    frames = batches[0]
    out = ta.augment_batch(frames, "cuda")
    torch.cuda.synchronize()
    staging, dev, d = out._vd3d_keepalive
    n, _, Ho, Wo = out.shape
    m, s = frames[0].mean, frames[0].std
    stream = torch.cuda.current_stream().cuda_stream
    vp = lambda a: a.ctypes.data

    def launch():
        _lib.call("vd3d_train_augment", d.data_ptr(), n, 3, Ho, Wo, vp(m), vp(s), out.data_ptr(), stream)

    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / launches
    read = sum((f.frame.shape[0] - f.crop_top) * f.frame.shape[1] * 3 for f in frames)
    nbytes = read + out.numel() * 4
    for fr in batches * 2:                                             # warm-up of the staging path
        ta.augment_batch(fr, "cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for fr in batches * 4:
        ta.augment_batch(fr, "cuda")
    torch.cuda.synchronize()
    batch_ms = (time.perf_counter() - t0) * 1e3 / (4 * len(batches))
    return {"images_per_batch": n, "output": [Ho, Wo], "host_ms_per_sample": round(host_ms, 3), "kernel_ms_per_batch": round(kernel_ms, 4),
            "kernel_bytes": nbytes, "kernel_GB_per_s": round(nbytes / kernel_ms / 1e6, 1),
            "kernel_share_of_hbm": round(nbytes / kernel_ms / 1e-3 / HBM_BYTES_PER_S, 3),
            "augment_batch_ms": round(batch_ms, 3)}


def train_step_arm(steps, warmup):
    """One train_stereo_detection step (reference Stereo3D, seeded synthetic weights, native anchor and disparity losses, batch 8 at
    288x1280) on a batch the reference dataset + collate_fn made from a synthetic KITTI tree of 375x1242 frames: with the reference's host
    augmentation (float images uploaded by the step) and with `plugin.install_train_augmentation_into_reference()` (uint8 staging
    uploaded and augmented on the GPU inside the step).  ms per step, host clock ending in a device synchronise."""
    import tempfile
    import refload
    sys.path.insert(0, os.path.join(ROOT, "tests", "workers"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from visualdet3d_b200 import plugin, synth
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    from make_golden_train_augment import edict
    from train_augment_plugin import write_tree
    from visualDet3D.data.kitti.dataset.stereo_dataset import KittiStereoDataset
    from visualDet3D.networks.utils import registry as ref
    tmp = tempfile.mkdtemp()
    obj = ["Car", "Pedestrian"]
    pm, ps = synth.synth_priors(16, 3, obj)
    synth.write_priors(tmp, pm, ps, obj)
    dcfg = refload.to_edict(dict(obj_types=obj, detector=synth.stereo3d_cfg(tmp, obj)))
    det = ref.DETECTOR_DICT["Stereo3D"](dcfg.detector)
    det.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in det.state_dict().items()}, 0), strict=False)
    det = det.cuda().train()
    plugin.install_loss_into_reference()
    plugin.install_disparity_loss_into_reference()
    opt = torch.optim.SGD(det.parameters(), lr=1e-6)
    pre = write_tree(tmp, [(H, W)] * BATCH)
    cfg = edict({"path": {"preprocessed_path": pre}, "obj_types": ["Car"], "optimizer": {"clipped_gradient_norm": 0.1},
                 "data": {"augmentation": {}, "train_augmentation": cases.LISTS["stereo3d"][0]}})

    def batch():
        ds = KittiStereoDataset(cfg, "training")
        np.random.seed(0)
        return KittiStereoDataset.collate_fn([ds[i] for i in range(BATCH)])

    def timed(data):
        fn = ref.PIPELINE_DICT["train_stereo_detection"]
        for _ in range(warmup):
            fn(data, det, opt, cfg=cfg)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn(data, det, opt, cfg=cfg)
        torch.cuda.synchronize()
        return round((time.perf_counter() - t0) * 1e3 / steps, 2)

    off = timed(batch())
    plugin.install_train_augmentation_into_reference()
    on = timed(batch())
    return {"train_step_ms_host_augmentation": off, "train_step_ms_gpu_augmentation": on, "batch": BATCH}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=32)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the GPU arm needs a CUDA device"
    res = {"card": card()}
    for cfg, name in CONFIGS.items():
        r = gpu_arm(name, a.samples, a.launches)
        r.update(reference_arm(name, a.samples, a.workers))
        res[cfg] = r
    res["train_stereo_detection"] = train_step_arm(a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
