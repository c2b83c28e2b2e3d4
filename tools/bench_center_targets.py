"""Time the KM3D / MonoFlex training targets: the reference's `_build_target` + collate_fn on the host against the GPU form
(visualdet3d_b200/center_targets.py: `DeferredTargetBatch.to_device`, two launches per batch), at 384x1280 with three classes:
  km3d:     batch 32 (KM3D_example's batch size), 9 keypoints;
  monoflex: batch 8, 10 keypoints;
each with KITTI-like object counts (4-12 per image) and at the 32-object cap.

Reports, per configuration:
  * the kernel time per batch (both launches) from CUDA events over `--launches` back-to-back batches after warm-up, and the bytes the
    kernels write (every target array, heatmaps included, plus the splat list) over that time;
  * to_device per batch (pinned staging upload, allocation, both launches; host clock ending in a device synchronise);
  * the reference's `_build_target` per sample and `_build_target` + collate_fn per batch on one host core, when the reference package is
    importable.
Prints one JSON line with the card's name, power limit and max SM clock; writes nothing.

    python tools/bench_center_targets.py [--launches 200] [--host-batches 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402
import center_targets_cases as cases  # noqa: E402
from bench_common import card  # noqa: E402
from visualdet3d_b200 import _lib  # noqa: E402
from visualdet3d_b200 import center_targets as ct  # noqa: E402

H, W, C = 384, 1280, 3
CONFIGS = {"km3d": (ct.MODE_KM3D, 32), "monoflex": (ct.MODE_MONOFLEX, 8)}


def label_sets(B, cap, seed):
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(B):
        n = 32 if cap else int(rng.randint(4, 13))
        out.append([cases.Obj(cases.random_obj(rng, cases.P2_KITTI, H, W), int(rng.randint(C))) for _ in range(n)])
    return out


def deferred(mode, labels):
    return [ct.DeferredTargets.build((H, W, 3), cases.P2_KITTI, objs, [cases.OBJ_TYPES.index(o.type) for o in objs], C, mode)
            for objs in labels]


def gpu_arm(mode, labels, launches):
    batch = ct.DeferredTargetBatch(deferred(mode, labels)).pin_memory()
    B = len(labels)
    outs = batch.to_device("cuda")
    recs = batch.staging.cuda()
    splats = torch.empty(B * int(_lib.load().vd3d_center_targets_splat_bytes()), dtype=torch.uint8, device="cuda")
    slots = [outs.get(key) for key, _, _ in ct._SLOTS]
    ptrs = (ct.ctypes.c_void_p * len(slots))(*[t.data_ptr() if t is not None else None for t in slots])
    stream = torch.cuda.current_stream().cuda_stream

    def launch():
        _lib.call("vd3d_center_targets", recs.data_ptr(), B, mode, H, W, C, ptrs, splats.data_ptr(), stream)

    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / launches
    written = sum(t.numel() * t.element_size() for t in slots if t is not None) + splats.numel()
    for _ in range(5):
        batch.to_device("cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(50):
        batch.to_device("cuda")
    torch.cuda.synchronize()
    to_device_ms = (time.perf_counter() - t0) * 1e3 / 50
    return {"kernel_ms_per_batch": round(kernel_ms, 4), "bytes_written": written,
            "write_GBps": round(written / (kernel_ms * 1e-3) / 1e9, 1), "to_device_ms_per_batch": round(to_device_ms, 3)}


def host_arm(mode, labels, batches):
    import refload
    if not refload.available():
        return None
    import pickle
    import tempfile
    refload.load_reference()
    from visualDet3D.data.kitti.dataset.KM3D_dataset import KittiMonoFlexDataset, KittiRTM3DDataset
    tmp = tempfile.mkdtemp()
    os.makedirs(os.path.join(tmp, "training"))
    with open(os.path.join(tmp, "training", "imdb.pkl"), "wb") as f:
        pickle.dump([], f)
    cfg = refload.EasyDict({"path": {"preprocessed_path": tmp}, "obj_types": cases.OBJ_TYPES,
                            "data": {"train_augmentation": [], "test_augmentation": []}})
    ds = (KittiMonoFlexDataset if mode == ct.MODE_MONOFLEX else KittiRTM3DDataset)(cfg, "training")
    image = np.zeros((H, W, 3), np.float32)
    torch.set_num_threads(1)
    t_build = t_all = 0.0
    for _ in range(batches):
        t0 = time.perf_counter()
        items = [{"image": image, "calib": cases.P2_KITTI, "label": ds._build_target(image, cases.P2_KITTI.copy(), objs)} for objs in labels]
        t1 = time.perf_counter()
        ds.collate_fn(items)
        t2 = time.perf_counter()
        t_build += t1 - t0
        t_all += t2 - t0
    return {"build_target_ms_per_sample": round(t_build * 1e3 / batches / len(labels), 3),
            "build_target_plus_collate_ms_per_batch": round(t_all * 1e3 / batches, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--host-batches", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_center_targets needs a CUDA device")
    res = {"card": card(), "size": [H, W], "classes": C}
    runs = [(f"{name}_{tag}", mode, label_sets(B, cap, seed=B + cap)) for name, (mode, B) in CONFIGS.items()
            for tag, cap in (("kitti", False), ("cap32", True))]
    for key, mode, labels in runs:
        res[key] = {"batch": len(labels), "objects": sum(len(x) for x in labels), **gpu_arm(mode, labels, a.launches)}
    for key, mode, labels in runs:           # after every GPU arm: the reference's CPU import turns torch.cuda.synchronize into a no-op
        res[key]["host_reference_one_core"] = host_arm(mode, labels, a.host_batches)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
