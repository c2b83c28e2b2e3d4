"""Golden vectors for visualdet3d_b200/kitti_eval.py from the UNMODIFIED reference evaluator (R/evaluator/kitti/evaluate.py) run on the
host through oracle/refload.py (numba CPU jit; its rotated-IoU kernel runs in the numba CUDA simulator).
python tests/golden/make_golden_kitti_eval.py  ->  tests/golden/kitti_eval.npz

Each case is a seeded synthetic KITTI label / result set; its text goes into the npz, so the tests need nothing else.  Stored per case:
the result string per class, precision / thresholds / orientation of each metric's eval_class, the per-image [3][dt][gt] overlaps, the
parsed annos, and `margin`.  The simulator's BEV / 3-D overlaps mix float64 into the float32 algorithm, so a device computes them
slightly differently: an image is redrawn while any BEV / 3-D overlap lies within MARGIN of a threshold (0.25, 0.5, 0.7) or two
above-threshold overlaps of one ground truth lie within MARGIN of each other.  Every matching decision then agrees on both sides.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
import refload  # noqa: E402

MARGIN = 1e-4
THRESHOLDS = (0.25, 0.5, 0.7)
DIMS = {"Car": (3.9, 1.55, 1.65), "Van": (5.0, 2.1, 1.9), "Pedestrian": (0.85, 1.75, 0.65), "Person_sitting": (0.8, 1.2, 0.6),
        "Cyclist": (1.75, 1.75, 0.6)}                                     # l, h, w
ANNO_KEYS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")


def gt_object(rng, name):
    if name == "DontCare":
        x1, y1 = rng.uniform(0, 1100), rng.uniform(120, 250)
        return dict(name=name, trunc=-1.0, occ=-1, alpha=-10.0, bbox=(x1, y1, x1 + rng.uniform(10, 80), y1 + rng.uniform(8, 40)),
                    dims=(-1.0, -1.0, -1.0), loc=(-1000.0, -1000.0, -1000.0), ry=-10.0)
    l, h, w = (d * rng.uniform(0.85, 1.15) for d in DIMS[name])
    z = rng.uniform(4, 60)
    x = rng.uniform(-0.5, 0.5) * z
    y = rng.uniform(1.4, 2.0)
    ry = rng.uniform(-np.pi, np.pi)
    cx = 720 * x / z + 610
    hh = 720 * h / z * rng.uniform(0.9, 1.1)          # 2-D heights from ~12 to ~300 px: both sides of 25 and 40
    ww = 720 * max(l, w) / z * rng.uniform(0.5, 1.0)
    y2 = 720 * y / z + 175
    return dict(name=name, trunc=float(rng.choice([0.0, 0.0, 0.1, 0.2, 0.4, 0.6])), occ=int(rng.choice([0, 0, 1, 2, 3])),
                alpha=float(np.arctan2(-x, z) + ry), bbox=(cx - ww / 2, y2 - hh, cx + ww / 2, y2), dims=(l, h, w), loc=(x, y, z), ry=ry)


def label_line(o):
    b, (l, h, w), (x, y, z) = o["bbox"], o["dims"], o["loc"]
    return (f"{o['name']} {o['trunc']:.2f} {o['occ']} {o['alpha']:.2f} {b[0]:.2f} {b[1]:.2f} {b[2]:.2f} {b[3]:.2f} "
            f"{h:.2f} {w:.2f} {l:.2f} {x:.2f} {y:.2f} {z:.2f} {o['ry']:.2f}")


def result_line(name, alpha, bbox, dims, loc, ry, score):
    """The format of the reference's write_result_to_file (data/kitti/utils.py:195-199)."""
    l, h, w = dims
    return ('{} -1 -1 {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {:.6f} {} \n').format(
        name, alpha, *bbox, h, w, l, *loc, ry, score)


def detections(rng, gts, two_d, names):
    out = []

    def emit(name, o, jit):
        b = np.array(o["bbox"]) + rng.normal(0, jit, 4) * (o["bbox"][3] - o["bbox"][1] + 5)
        dims = tuple(np.array(o["dims"]) * rng.uniform(0.9, 1.1, 3))
        loc = tuple(np.array(o["loc"]) + rng.normal(0, 0.3, 3) * np.array([1, 0.3, 1]) * (1 + o["loc"][2] / 40))
        ry = o["ry"] + rng.normal(0, 0.25)
        alpha = o["alpha"] + rng.normal(0, 0.25)
        if two_d:
            alpha, dims, loc, ry = -10, (-1, -1, -1), (-1000, -1000, -1000), -10
        out.append(result_line(name, alpha, b, dims, loc, ry, round(float(rng.uniform(0.05, 1.0)), 4)))

    for o in gts:
        if o["name"] == "DontCare" or rng.uniform() < 0.15:
            continue
        name = {"Van": "Car", "Person_sitting": "Pedestrian"}.get(o["name"], o["name"]) if rng.uniform() < 0.3 else o["name"]
        emit(name, o, 0.06)
        if rng.uniform() < 0.25:                        # duplicate
            emit(name, o, 0.12)
    for _ in range(rng.randint(0, 5)):                  # false positives, some below the 25 px minimum
        emit(str(rng.choice(names)), gt_object(rng, str(rng.choice(["Car", "Pedestrian", "Cyclist"]))), 0.05)
    rng.shuffle(out)
    return "".join(out)


def anno_boxes(a):
    bev = np.concatenate([a["location"][:, [0, 2]], a["dimensions"][:, [0, 2]], a["rotation_y"][:, None]], 1)
    d3 = np.concatenate([a["location"], a["dimensions"], a["rotation_y"][:, None]], 1)
    return bev, d3


def bev_3d_overlaps(E, gt, dt):
    """The reference's BEV / 3-D overlaps of one image, [dt][gt], as eval_class computes them (arguments swapped as it swaps them)."""
    gb, g3 = anno_boxes(gt)
    db, d3 = anno_boxes(dt)
    if len(gb) == 0 or len(db) == 0:
        return np.zeros((2, len(db), len(gb)))
    return np.stack([E.bev_box_overlap(db, gb).astype(np.float64), E.d3_box_overlap(d3, g3).astype(np.float64)])


def margin_of(ovs):
    """Smallest distance of a BEV / 3-D overlap to a threshold, or between two above-threshold overlaps of one ground truth."""
    m = np.inf
    for ov in ovs:                                      # [2][dt][gt]
        if ov.size == 0:
            continue
        for t in THRESHOLDS:
            m = min(m, float(np.abs(ov - t).min()))
        for col in ov.transpose(0, 2, 1).reshape(-1, ov.shape[1]):
            v = np.sort(col[col > min(THRESHOLDS)])
            if len(v) > 1:
                m = min(m, float(np.diff(v).min()))
    return m


def make_case(E, KC, seed, n_img, two_d=False, no_cyclist_gt=False, dontcare=True):
    rng = np.random.RandomState(seed)
    ids = np.sort(rng.choice(np.arange(8000), n_img, replace=False))
    classes = ["Car", "Car", "Car", "Van", "Pedestrian", "Pedestrian", "Person_sitting", "Cyclist", "Cyclist"]
    if no_cyclist_gt:
        classes = [c for c in classes if c != "Cyclist"]
    if dontcare:
        classes.append("DontCare")
    labels, results = [], []
    tmp = tempfile.mkdtemp()
    for i in range(n_img):
        n_obj = 0 if i % 11 == 3 else rng.randint(1, 13)
        gts = [gt_object(rng, str(rng.choice(classes))) for _ in range(n_obj)]
        label = "".join(label_line(o) + "\n" for o in gts)
        gt_anno = parse(KC, tmp, label)
        for _ in range(100):
            res = "" if i % 13 == 5 else detections(rng, gts, two_d, ["Car", "Pedestrian", "Cyclist"])
            if margin_of([bev_3d_overlaps(E, gt_anno, parse(KC, tmp, res))]) > MARGIN:
                break
        else:
            raise RuntimeError(f"seed {seed} image {i}: no draw with a margin above {MARGIN}")
        labels.append(label)
        results.append(res)
    return ids, labels, results


def parse(KC, tmp, text):
    p = os.path.join(tmp, "x.txt")
    with open(p, "w") as f:
        f.write(text)
    return KC.get_label_anno(p)


def write_set(root, ids, labels, results):
    lab, res = os.path.join(root, "label_2"), os.path.join(root, "data")
    os.makedirs(lab)
    os.makedirs(res)
    for i, l, r in zip(ids, labels, results):
        with open(os.path.join(lab, f"{i:06d}.txt"), "w") as f:
            f.write(l)
        with open(os.path.join(res, f"{i:06d}.txt"), "w") as f:
            f.write(r)
    split = os.path.join(root, "val.txt")
    with open(split, "w") as f:
        f.write("".join(f"{i:06d}\n" for i in ids))
    return lab, res, split


def run_reference(E, KE, KC, ids, labels, results, classes, one_part):
    captured, ious = [], {}
    do_eval_v3, calc = E.do_eval_v3, E.calculate_iou_partly
    split_parts = E.get_split_parts

    def cap_eval(*a, **k):
        r = do_eval_v3(*a, **k)
        captured.append(r)
        return r

    def cap_iou(dt_annos, gt_annos, metric, *a, **k):
        r = calc(dt_annos, gt_annos, metric, *a, **k)
        ious.setdefault(metric, r[0])
        return r

    E.do_eval_v3, E.calculate_iou_partly = cap_eval, cap_iou
    if one_part:     # the split only groups the overlap computation; with fewer than 50 images its parts are empty
        E.get_split_parts = lambda num, num_part: [num]
    try:
        with tempfile.TemporaryDirectory() as root:
            lab, res, split = write_set(root, ids, labels, results)
            texts = KE.evaluate(label_path=lab, result_path=res, label_split_file=split, current_classes=list(classes), gpu=0)
            gt_annos = KC.get_label_annos(lab, [int(i) for i in ids])
            dt_annos = KC.get_label_annos(res)
    finally:
        E.do_eval_v3, E.calculate_iou_partly, E.get_split_parts = do_eval_v3, calc, split_parts
    return texts, captured, ious, gt_annos, dt_annos


def store_case(out, name, ids, labels, results, classes, texts, captured, ious, gt_annos, dt_annos):
    """One case under the keys `name/...` (what tests/test_kitti_eval_cpu.py::write_case and the GPU tests read); returns (ng, nd)."""
    p = f"{name}/"
    out.update({p + "ids": ids, p + "label_text": np.array(labels), p + "result_text": np.array(results),
                p + "classes": np.array(classes, dtype=np.int64), p + "texts": np.array(texts)})
    for m in ("bbox", "bev", "3d"):
        for key in ("precision", "thresholds", "orientation"):
            if key == "orientation" and m != "bbox":
                continue
            out[p + f"{m}_{key}"] = np.concatenate([r[m][key] for r in captured], 0)
    ng = np.array([len(a["name"]) for a in gt_annos])
    nd = np.array([len(a["name"]) for a in dt_annos])
    out[p + "ng"], out[p + "nd"] = ng, nd
    out[p + "overlaps"] = np.stack([np.concatenate([o.reshape(-1) for o in ious[m]]) for m in range(3)])
    for who, annos in (("gt", gt_annos), ("dt", dt_annos)):
        out[p + f"{who}_name"] = np.array([n for a in annos for n in a["name"]], dtype=str)   # an empty file parses to float64
        for k in ANNO_KEYS[1:]:
            out[p + f"{who}_{k}"] = np.concatenate([a[k] for a in annos], 0)
    per_image = [np.stack([ious[1][i], ious[2][i]]) for i in range(len(ids))]
    out[p + "margin"] = np.float64(margin_of(per_image))
    return ng, nd


def main():
    refload.load_reference()
    import visualDet3D.evaluator.kitti.eval as E
    import visualDet3D.evaluator.kitti.evaluate as KE
    import visualDet3D.evaluator.kitti.kitti_common as KC
    cases = {
        "mixed": dict(seed=11, n_img=120, classes=(0, 1, 2)),
        "bbox2d": dict(seed=12, n_img=60, classes=(0, 1, 2), two_d=True, dontcare=False),
        "small": dict(seed=13, n_img=40, classes=(0, 1, 2), no_cyclist_gt=True),
    }
    from visualDet3D.evaluator.kitti.rotate_iou import rotate_iou_gpu_eval
    rng = np.random.RandomState(7)                      # rotate_iou_gpu_eval alone: overlapping rotated boxes, all four criteria
    boxes = np.concatenate([rng.uniform(-3, 3, (48, 2)), rng.uniform(0.5, 4.5, (48, 2)), rng.uniform(-np.pi, np.pi, (48, 1))], 1)
    qboxes = np.concatenate([rng.uniform(-3, 3, (40, 2)), rng.uniform(0.5, 4.5, (40, 2)), rng.uniform(-np.pi, np.pi, (40, 1))], 1)
    out = {"riou/boxes": boxes.astype(np.float32), "riou/qboxes": qboxes.astype(np.float32)}
    for crit in (-1, 0, 1, 2):
        out[f"riou/crit{crit}"] = rotate_iou_gpu_eval(boxes, qboxes, crit)
    for name, c in cases.items():
        ids, labels, results = make_case(E, KC, c["seed"], c["n_img"], c.get("two_d", False), c.get("no_cyclist_gt", False),
                                         c.get("dontcare", True))
        texts, captured, ious, gt_annos, dt_annos = run_reference(E, KE, KC, ids, labels, results, c["classes"], c["n_img"] < 50)
        ng, nd = store_case(out, name, ids, labels, results, c["classes"], texts, captured, ious, gt_annos, dt_annos)
        print(f"{name}: {len(ids)} images, {ng.sum()} gt, {nd.sum()} dt, margin {float(out[name + '/margin']):.3g}")
        print(texts[0])
    np.savez_compressed(os.path.join(HERE, "kitti_eval.npz"), **out)


if __name__ == "__main__":
    main()
