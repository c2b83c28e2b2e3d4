"""Timing of the det_precompute anchor priors on the GPU.  Prints one JSON line.

  (a) kernel: one batch of 64 frames at Stereo3D's 288x1280 table (69,120 anchors, 48 bins, Car / Pedestrian) with KITTI-like box
      counts (Car 0-12, Pedestrian 0-4 per frame).  `*_kernels_ms`: the device durations of prior_iou_kernel + prior_walk_kernel from
      torch.profiler, per batch.  `*_entry_ms`: CUDA events around the C entry alone (offsets copy, key memset, both launches and their
      host-side enqueue; the Python checks and the workspace allocation are outside), median over the repeats.
  (b) end to end: frames/s of `python -m visualdet3d_b200.det_precompute --split=train` (training split only, the priors included) against
      the unmodified reference scripts/imdb_precompute_3d.py read_one_split on the same GPU (its copy under oracle/_ref/scripts; skipped
      when absent), over a constructed KITTI tree of --frames frames (tests/det_precompute_cases.write_tree) in a temporary directory.

    python tools/bench_det_precompute.py [--frames 200] [--repeats 50]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]


def kernel_times(repeats):
    import torch
    from visualdet3d_b200 import anchor_prior as ap
    from visualdet3d_b200.anchors import grid_anchors
    cfg = dict(pyramid_levels=[4], strides=[16], sizes=[24], ratios=np.array([0.5, 1, 2.0]), scales=np.array([2 ** (i / 4.0) for i in range(16)]))
    acc = ap.AnchorPriorAccumulator(cfg, (288, 1280), ["Car", "Pedestrian"], 0.5, "cuda")
    anchors, order, start = acc.table((288, 1280))
    rng = np.random.RandomState(0)
    a32 = anchors.cpu().numpy()
    counts = np.stack([rng.randint(0, 13, 64), rng.randint(0, 5, 64)], axis=1).reshape(-1)
    off = np.zeros(len(counts) + 1, np.int32)
    off[1:] = np.cumsum(counts)
    boxes = (a32[rng.randint(0, len(a32), off[-1])] + rng.uniform(-6, 6, (off[-1], 4))).astype(np.float32)
    gt3 = np.stack([rng.uniform(5, 60, off[-1]), rng.uniform(-1, 1, off[-1]), rng.uniform(-1, 1, off[-1])], axis=1)
    bx, g = torch.from_numpy(boxes).cuda(), torch.from_numpy(gt3).cuda()
    st = ap.PriorState(2, 48, "cuda")
    out = {}
    for name, b in (("f32", bx), ("f64", bx.double())):
        call = ap.prepare(st, anchors, order, start, off, b, g, 0.5)   # checks and workspace outside the timed window
        for _ in range(5):
            call()
        ts = []
        for _ in range(repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        out[f"batch64_{name}_entry_ms"] = float(np.median(ts))
        # the two kernels alone: device durations from the profiler, per batch
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(repeats):
                call()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            if "prior_iou_kernel" in ev.key or "prior_walk_kernel" in ev.key:
                key = "iou" if "prior_iou" in ev.key else "walk"
                per[key] = per.get(key, 0.0) + ev.device_time_total / 1000.0
        for key, v in per.items():
            out[f"batch64_{name}_{key}_kernel_ms"] = v / repeats
        out[f"batch64_{name}_kernels_ms"] = sum(per.values()) / repeats
    out["positives_per_batch"] = int(st.numpy()["examine"].sum() // (2 * (5 + 2 * repeats)))
    out["boxes_per_batch"] = int(off[-1])
    return out


CLI = """import os, sys, time
ROOT, cfgp, mode = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
import refload
from visualdet3d_b200.ops import dcn, iou3d
refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
import torch
from visualDet3D.utils.utils import cfg_from_file
cfg = cfg_from_file(cfgp)
torch.zeros(1, device="cuda")
if mode == "ours":
    from visualdet3d_b200 import det_precompute as m
else:
    import make_golden_det_precompute as mg
    m, _ = mg.reference_scripts(os.path.join(ROOT, "oracle", "_ref", "scripts"), cpu=False)
tr, _ = m.process_train_val_file(cfg)
t0 = time.time()
m.read_one_split(cfg, tr, cfg.path.data_path, {"calib": True, "image": True, "label": True, "velodyne": False}, 'training', 10 ** 9)
torch.cuda.synchronize()
print("FPS", len(tr) / (time.time() - t0))
"""


def cli_fps(frames):
    import det_precompute_cases as dc
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        raw, split = dc.write_tree(tmp, n_frames=frames)
        with open(os.path.join(split, "train.txt"), "w") as f:              # time the whole tree as the training split
            f.write("".join("%06d\n" % i for i in range(frames)))
        modes = ["ours"] + (["reference"] if os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "scripts")) else [])
        for mode in modes:
            cfgp = dc.write_config("stereo3d", os.path.join(tmp, mode), raw, split)
            r = subprocess.run([sys.executable, "-c", CLI, ROOT, cfgp, mode], capture_output=True, text=True, timeout=3000)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("FPS")]
            out[f"cli_{mode}_frames_per_s"] = float(line[-1].split()[1]) if line else r.stderr[-500:]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=50)
    a = ap.parse_args()
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": q or torch.cuda.get_device_name(0), "host_cores": os.cpu_count()}
    res.update(kernel_times(a.repeats))
    res.update(cli_fps(a.frames))
    res["frames"] = a.frames
    print(json.dumps(res))


if __name__ == "__main__":
    main()
