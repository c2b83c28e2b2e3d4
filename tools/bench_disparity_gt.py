"""Time Stereo3D's disparity ground truth (visualdet3d_b200/disparity_gt.py, csrc/disparity_gt.cu) at the reference's precompute size,
288x1280 (Stereo3D_example's test augmentation):
  * bm_targets per pair at batch 8 (float32 network input -> the written uint16 map), and stereo_bm alone (uint8 grey in), from CUDA
    events over --launches batches after warm-up;
  * velo_targets per frame of a 120k-point cloud, likewise;
  * cv2.StereoBM_create(192, 25).compute on the host cores, at the best of the thread counts tried, on the same pairs;
  * the precompute CLI end to end (PNG decode, the reference's test augmentation, device maps, PNG writes) in frames per second over a
    generated KITTI tree of --frames frames, when the reference package is importable;
  * a check that the device maps equal cv2's at the timed size.
Prints one JSON line with the card's name and power limit.  Scratch files go to a temporary directory.

    python tools/bench_disparity_gt.py [--launches 50] [--frames 32]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import cv2  # noqa: E402
import torch  # noqa: E402
import disparity_gt_cases as dc  # noqa: E402
from bench_common import card  # noqa: E402
from visualdet3d_b200 import disparity_gt as dg  # noqa: E402

H, W, B = 288, 1280, 8


def event_ms(fn, launches):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def cv2_ms(L, R):
    best = None
    m = cv2.StereoBM_create(192, 25)
    for threads in (1, 2, 4, 8, 16, os.cpu_count() or 1):
        cv2.setNumThreads(threads)
        m.compute(L[0], R[0])
        t = time.perf_counter()
        for b in range(len(L)):
            m.compute(L[b], R[b])
        ms = (time.perf_counter() - t) * 1e3 / len(L)
        if best is None or ms < best[0]:
            best = (ms, threads)
    return best


CLI = """import os, runpy, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "oracle")]
import refload
from visualdet3d_b200.ops import dcn, iou3d
refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
sys.argv = ["disparity_precompute"] + sys.argv[2:]
runpy.run_module("visualdet3d_b200.disparity_precompute", run_name="__main__")
"""


def cli_fps(frames, pc):
    import refload
    if not refload.available():
        return None
    with tempfile.TemporaryDirectory() as tmp:
        cfg = dc.write_tree(tmp, sizes=[(375, 1242)] * frames, n_points=120000)
        t = time.perf_counter()
        r = subprocess.run([sys.executable, "-c", CLI, ROOT, f"--config={cfg}", f"--use_point_cloud={pc}"], capture_output=True, text=True,
                           cwd=tmp)
        wall = time.perf_counter() - t
        if r.returncode != 0:
            raise RuntimeError(r.stderr[-3000:])
        # the process's own report covers the loop only (imports and CUDA start-up excluded)
        last = [line for line in r.stdout.splitlines() if "frames/s" in line][-1]
        return {"loop_frames_per_s": float(last.split(",")[1].split()[0]), "process_wall_s": round(wall, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--frames", type=int, default=32)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    cases = [dc.banded(100 + b, H, W, dc._bands(H, [5 + 20 * b, 60 + 15 * b, 150])) for b in range(B)]
    L = np.stack([c[0] for c in cases])
    R = np.stack([c[1] for c in cases])
    Lf = np.stack([((np.repeat(l[..., None], 3, 2) / 255.0 - dc.MEAN) / dc.STD).astype(np.float32) for l in L])
    Rf = np.stack([((np.repeat(r[..., None], 3, 2) / 255.0 - dc.MEAN) / dc.STD).astype(np.float32) for r in R])
    gl, gr = torch.from_numpy(L).cuda(), torch.from_numpy(R).cuda()
    fl, fr = torch.from_numpy(Lf).cuda(), torch.from_numpy(Rf).cuda()
    targets_ms = event_ms(lambda: dg.bm_targets(fl, fr, dc.MEAN, dc.STD), a.launches)
    bm_ms = event_ms(lambda: dg.stereo_bm(gl, gr), a.launches)
    pts = torch.from_numpy(dc.velo_cases()[1]["points"]).cuda()
    velo_ms = event_ms(lambda: dg.velo_targets(pts, dc.R0, dc.TR, dc.P2, dc.BASELINE, H, W), a.launches)

    # the float frames' reference: the script's denorm (which truncates, so it need not give L back) + cvtColor, then cv2
    import stereo_bm as sb
    m = cv2.StereoBM_create(192, 25)
    ref = np.stack([m.compute(L[b], R[b]) for b in range(B)])
    grey = lambda f: cv2.cvtColor(sb.denorm(f, dc.MEAN, dc.STD), cv2.COLOR_BGR2GRAY)
    ref_f = [m.compute(grey(Lf[b]), grey(Rf[b])) for b in range(B)]
    maps = dg.bm_targets(fl, fr, dc.MEAN, dc.STD).cpu().numpy()
    equal = bool(np.array_equal(dg.stereo_bm(gl, gr).cpu().numpy(), ref)) and \
        all(np.array_equal(maps[b], sb.block_max(ref_f[b])) for b in range(B))
    cv_ms, cv_threads = cv2_ms(L, R)
    out = {"metric": "disparity_gt", "size": [H, W], "batch": B,
           "bm_targets_ms_per_pair": round(targets_ms / B, 4), "stereo_bm_ms_per_pair": round(bm_ms / B, 4),
           "velo_targets_ms_per_frame_120k": round(velo_ms, 4),
           "cv2_compute_ms_per_pair": round(cv_ms, 2), "cv2_threads": cv_threads, "cv2_host_cores": os.cpu_count(),
           "device_equals_cv2": equal,
           "cli_bm": cli_fps(a.frames, "False"), "cli_velo": cli_fps(a.frames, "True"), "card": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
