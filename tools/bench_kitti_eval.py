"""Time the native KITTI evaluator (visualdet3d_b200/kitti_eval.py) on a seeded KITTI-val-sized set, and the reference evaluator on the
same files where it can run with a real numba CUDA device.

    python tools/bench_kitti_eval.py [--images 3769] [--iters 5] [--no-reference] [--coco]

Writes the label / result files to a temporary directory and prints one JSON line: the wall time of evaluate() split into parse /
device / format, the device part alone from CUDA events after a warm-up, the card and its power limit, and the reference's wall time
with a check that its strings are equal ("not measured" where the reference or numba's CUDA target is missing).  --coco adds "coco":
the same split and CUDA-event timing for get_coco_eval_result's device part (one vd3d_kitti_eval call per class over ten min-overlap
rows) next to the official evaluation's."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import textwrap
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from visualdet3d_b200 import kitti_eval  # noqa: E402

CLASSES = ["Car"] * 8 + ["Van", "Pedestrian", "Pedestrian", "Person_sitting", "Cyclist", "DontCare", "DontCare"]


def write_set(root, n_img, seed):
    """KITTI-like object counts (about 7 labelled objects per image) and 20-50 scored detections per image."""
    rng = np.random.RandomState(seed)
    lab, res = os.path.join(root, "label_2"), os.path.join(root, "data")
    os.makedirs(lab)
    os.makedirs(res)
    ids = list(range(n_img))
    for i in ids:
        n = rng.poisson(7)
        z = rng.uniform(5, 70, n)
        x = rng.uniform(-0.5, 0.5, n) * z
        y = rng.uniform(1.4, 2.0, n)
        lhw = np.stack([rng.uniform(0.7, 5.0, n), rng.uniform(1.2, 2.2, n), rng.uniform(0.5, 2.0, n)], 1)
        ry = rng.uniform(-np.pi, np.pi, n)
        cx, y2 = 720 * x / z + 610, 720 * y / z + 175
        hh, ww = 720 * lhw[:, 1] / z, 720 * lhw[:, 0] / z * 0.8
        names = rng.choice(CLASSES, n)
        lines = []
        for k in range(n):
            lines.append(f"{names[k]} {rng.choice([0.0, 0.2, 0.5]):.2f} {rng.randint(0, 3)} {ry[k] - np.arctan2(x[k], z[k]):.2f} "
                         f"{cx[k] - ww[k] / 2:.2f} {y2[k] - hh[k]:.2f} {cx[k] + ww[k] / 2:.2f} {y2[k]:.2f} "
                         f"{lhw[k, 1]:.2f} {lhw[k, 2]:.2f} {lhw[k, 0]:.2f} {x[k]:.2f} {y[k]:.2f} {z[k]:.2f} {ry[k]:.2f}\n")
        with open(os.path.join(lab, f"{i:06d}.txt"), "w") as f:
            f.write("".join(lines))
        m = rng.randint(20, 51)
        src = rng.randint(0, max(n, 1), m)
        real = (rng.uniform(size=m) < 0.5) & (n > 0)
        dets = []
        for j in range(m):
            if real[j]:
                k = src[j]
                b = np.array([cx[k] - ww[k] / 2, y2[k] - hh[k], cx[k] + ww[k] / 2, y2[k]]) + rng.normal(0, 0.08 * hh[k] + 1, 4)
                loc = np.array([x[k], y[k], z[k]]) + rng.normal(0, 0.4, 3)
                d, r, name = lhw[k] * rng.uniform(0.9, 1.1, 3), ry[k] + rng.normal(0, 0.3), names[k] if names[k] != "DontCare" else "Car"
            else:
                zz = rng.uniform(5, 70)
                loc = np.array([rng.uniform(-0.5, 0.5) * zz, 1.7, zz])
                u, v = 720 * loc[0] / zz + 610, 720 * 1.7 / zz + 175
                b = np.array([u - 40, v - 50, u + 40, v]) * rng.uniform(0.5, 1.5)
                d, r, name = np.array([3.9, 1.5, 1.6]), rng.uniform(-np.pi, np.pi), rng.choice(["Car", "Pedestrian", "Cyclist"])
            dets.append(('{} -1 -1 {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {} \n').format(
                name, r - np.arctan2(loc[0], loc[2]), *b, d[1], d[2], d[0], *loc, r, round(float(rng.beta(2, 2)), 4)))
        with open(os.path.join(res, f"{i:06d}.txt"), "w") as f:
            f.write("".join(dets))
    split = os.path.join(root, "val.txt")
    with open(split, "w") as f:
        f.write("".join(f"{i:06d}\n" for i in ids))
    return lab, res, split


def device_part(gt_annos, dt_annos, classes, min_overlaps_of, format_result, iters):
    """One DeviceEval per class (pack, upload, run, download) and its text, timed; then the launches alone with CUDA events."""
    t_dev = t_fmt = 0.0
    texts, evals = [], []
    for c in classes:
        cls = kitti_eval._class_indices(c)
        aos = kitti_eval._compute_aos(dt_annos)
        ta = time.perf_counter()
        ev = kitti_eval.DeviceEval(gt_annos, dt_annos, cls, min_overlaps_of(cls), aos)
        metrics = ev.run().collect()
        tb = time.perf_counter()
        texts.append(format_result(metrics, cls, aos))
        tc = time.perf_counter()
        t_dev += tb - ta
        t_fmt += tc - tb
        evals.append(ev)
    for ev in evals:                       # warm-up done above; now the launches alone
        ev.run()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        for ev in evals:
            ev.run()
    end.record()
    end.synchronize()
    return texts, t_dev, t_fmt, start.elapsed_time(end) / iters


def native(lab, res, split, classes, iters, coco):
    """evaluate() step by step (the same calls it makes), timed per stage; then the device part alone with CUDA events.  With coco,
    get_coco_eval_result's device part on the same parsed annos, timed the same way."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dt_annos = kitti_eval.get_label_annos(res)
    gt_annos = kitti_eval.get_label_annos(lab, kitti_eval._read_imageset_file(split))
    t1 = time.perf_counter()
    texts, t_dev, t_fmt, ev_ms = device_part(gt_annos, dt_annos, classes, lambda cls: kitti_eval.MIN_OVERLAPS[:, :, cls],
                                             kitti_eval.format_official_result, iters)
    assert texts == kitti_eval.evaluate(lab, res, split, classes, gpu=torch.cuda.current_device())
    out = {"parse_s": t1 - t0, "device_s": t_dev, "format_s": t_fmt, "total_s": t1 - t0 + t_dev + t_fmt,
           "device_events_ms": ev_ms, "n_gt": int(sum(len(a["name"]) for a in gt_annos)),
           "n_dt": int(sum(len(a["name"]) for a in dt_annos))}
    if coco:
        coco_texts, c_dev, c_fmt, c_ms = device_part(
            gt_annos, dt_annos, classes, lambda cls: kitti_eval.coco_min_overlaps(kitti_eval._coco_overlap_ranges(cls)),
            kitti_eval.format_coco_result, iters)
        assert coco_texts == [kitti_eval.get_coco_eval_result(gt_annos, dt_annos, c) for c in classes]
        out["coco"] = {"device_s": c_dev, "format_s": c_fmt, "device_events_ms": c_ms, "official_device_events_ms": ev_ms,
                       "min_overlap_rows": 10,
                       "reference": "not measured: its get_coco_eval_result raises TypeError on numpy >= 1.18 (np.linspace num as float64)"}
        texts = texts + coco_texts
    return texts, out


REF_CODE = """
import json, sys, time
sys.path[:0] = [{oracle!r}]
import refload
if not refload.available():
    print("REF_JSON " + json.dumps({{"status": "not measured: no reference package"}})); sys.exit(0)
refload.load_reference()
from numba import cuda
if not cuda.is_available():
    print("REF_JSON " + json.dumps({{"status": "not measured: no numba CUDA device"}})); sys.exit(0)
from visualDet3D.evaluator.kitti.evaluate import evaluate
t = time.perf_counter()
texts = evaluate({lab!r}, {res!r}, {split!r}, {classes!r}, gpu=0)
print("REF_JSON " + json.dumps({{"status": "ok", "wall_s": time.perf_counter() - t, "texts": texts}}))
"""


def reference(lab, res, split, classes, timeout):
    """The unmodified reference evaluate() with numba's real CUDA target, in its own process (importing the reference patches torch)."""
    code = textwrap.dedent(REF_CODE.format(oracle=os.path.join(ROOT, "oracle"), lab=lab, res=res, split=split, classes=classes))
    env = dict(os.environ, NUMBA_ENABLE_CUDASIM="0")
    try:
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    except subprocess.TimeoutExpired:
        return {"status": f"not measured: over {timeout} s"}
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("REF_JSON ")]
    if r.returncode != 0 or not lines:
        return {"status": "not measured: " + (r.stderr.strip().splitlines() or ["failed"])[-1][:200]}
    return json.loads(lines[-1][len("REF_JSON "):])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--reference-timeout", type=int, default=900)
    ap.add_argument("--coco", action="store_true", help="also time the COCO-style evaluation's device part")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_eval needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    classes = [0, 1, 2]
    with tempfile.TemporaryDirectory() as root:
        lab, res, split = write_set(root, args.images, args.seed)
        texts, out = native(lab, res, split, classes, args.iters, args.coco)
        ref = {"status": "not measured: --no-reference"} if args.no_reference else reference(lab, res, split, classes, args.reference_timeout)
    if "texts" in ref:
        ref["strings_equal"] = ref.pop("texts") == texts[:len(classes)]
    out.update({"images": args.images, "classes": classes, "gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown",
                "reference": ref})
    print(texts[0])
    if args.coco:
        print(texts[len(classes)])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
