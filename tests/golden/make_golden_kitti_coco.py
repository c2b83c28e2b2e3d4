"""Golden vectors for the COCO-style KITTI AP of visualdet3d_b200/kitti_eval.py from the UNMODIFIED reference evaluator
(R/evaluator/kitti/eval.py get_coco_eval_result, eval_class) run on the host through oracle/refload.py (numba CPU jit; its rotated-IoU
kernel runs in the numba CUDA simulator).
python tests/golden/make_golden_kitti_coco.py  ->  tests/golden/kitti_coco.npz

The reference's do_coco_style_eval passes the number of rows to np.linspace as a float64, which numpy >= 1.18 refuses; inside this
process only, np.linspace casts `num` to int.  That is the only shim.  Scenes are drawn as in make_golden_kitti_eval.py, with the same
margin-redraw rule, here around every min overlap either evaluation uses: the official 0.25 / 0.5 / 0.7 and the COCO rows.  Stored per
case: the label / result text, the classes, the reference's get_coco_eval_result text per class, and eval_class's precision /
thresholds (every metric) and orientation (bbox) over the ten rows of all the case's classes at once.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
sys.path.insert(0, HERE)
import refload  # noqa: E402
import make_golden_kitti_eval as mk  # noqa: E402

# eval.py:818-827, the class_to_range get_coco_eval_result uses: [first, last, number of] min overlaps per class
CLASS_TO_RANGE = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10], 3: [0.5, 0.95, 10], 4: [0.25, 0.7, 10],
                  5: [0.5, 0.95, 10], 6: [0.5, 0.95, 10], 7: [0.5, 0.95, 10]}
COCO_ROWS = np.concatenate([np.linspace(0.5, 0.95, 10), np.linspace(0.25, 0.7, 10)])
mk.THRESHOLDS = tuple(sorted(set((0.25, 0.5, 0.7)) | set(COCO_ROWS.tolist())))   # margin_of reads the module's THRESHOLDS


def _linspace_int_num(start, stop, num=50, *args, _linspace=np.linspace, **kwargs):
    return _linspace(start, stop, int(num), *args, **kwargs)


def make_case(E, KC, seed, n_img, two_d=False, cyclist_occluded=None):
    """make_golden_kitti_eval.make_case; cyclist_occluded sets every Cyclist's occlusion level (1: none in the easy difficulty).  2-D
    results get no DontCare labels: their placeholder 3-D boxes would overlap the DontCare placeholders at fixed values."""
    rng = np.random.RandomState(seed)
    ids = np.sort(rng.choice(np.arange(8000), n_img, replace=False))
    classes = ["Car", "Car", "Car", "Van", "Pedestrian", "Pedestrian", "Person_sitting", "Cyclist", "Cyclist"] + ([] if two_d else ["DontCare"])
    labels, results = [], []
    tmp = tempfile.mkdtemp()
    for i in range(n_img):
        n_obj = 0 if i % 11 == 3 else rng.randint(1, 13)                 # images without labels
        gts = [mk.gt_object(rng, str(rng.choice(classes))) for _ in range(n_obj)]
        if cyclist_occluded is not None:
            for o in gts:
                if o["name"] == "Cyclist":
                    o["occ"] = cyclist_occluded
        label = "".join(mk.label_line(o) + "\n" for o in gts)
        gt_anno = mk.parse(KC, tmp, label)
        for _ in range(100):
            res = "" if i % 13 == 5 else mk.detections(rng, gts, two_d, ["Car", "Pedestrian", "Cyclist"])   # images without detections
            if mk.margin_of([mk.bev_3d_overlaps(E, gt_anno, mk.parse(KC, tmp, res))]) > mk.MARGIN:
                break
        else:
            raise RuntimeError(f"seed {seed} image {i}: no draw with a margin above {mk.MARGIN}")
        labels.append(label)
        results.append(res)
    return ids, labels, results


def run_reference(E, KC, ids, labels, results, classes):
    split_parts = E.get_split_parts
    if len(ids) < 50:     # the split only groups the overlap computation; with fewer than 50 images its parts are empty
        E.get_split_parts = lambda num, num_part: [num]
    try:
        with tempfile.TemporaryDirectory() as root:
            lab, res, _ = mk.write_set(root, ids, labels, results)
            gt_annos = KC.get_label_annos(lab, [int(i) for i in ids])
            dt_annos = KC.get_label_annos(res)
        texts = [E.get_coco_eval_result(gt_annos, dt_annos, c) for c in classes]
        compute_aos = "aos  AP" in texts[0]
        overlap_ranges = np.zeros([3, 3, len(classes)])
        for i, c in enumerate(classes):
            overlap_ranges[:, :, i] = np.array(CLASS_TO_RANGE[c])[:, np.newaxis]
        min_overlaps = np.zeros([10, 3, len(classes)])                  # do_coco_style_eval's rows (np.linspace is the shim)
        for i in range(3):
            for j in range(len(classes)):
                min_overlaps[:, i, j] = np.linspace(*overlap_ranges[:, i, j])
        curves = {m: E.eval_class(gt_annos, dt_annos, list(classes), (0, 1, 2), m, min_overlaps, compute_aos and m == 0)
                  for m in range(3)}
    finally:
        E.get_split_parts = split_parts
    return texts, curves, min_overlaps, compute_aos, gt_annos, dt_annos


def main():
    np.linspace = _linspace_int_num
    refload.load_reference()
    import visualDet3D.evaluator.kitti.eval as E
    import visualDet3D.evaluator.kitti.kitti_common as KC
    cases = {
        "mixed": dict(seed=21, n_img=80, classes=(0, 1, 2)),
        "bbox2d": dict(seed=22, n_img=60, classes=(0, 1, 2), two_d=True),                # alpha = -10: no AOS line
        "occluded_cyclists": dict(seed=23, n_img=40, classes=(0, 1, 2), cyclist_occluded=1),   # no easy Cyclist ground truth
    }
    out = {}
    for name, c in cases.items():
        ids, labels, results = make_case(E, KC, c["seed"], c["n_img"], c.get("two_d", False), c.get("cyclist_occluded"))
        texts, curves, min_overlaps, compute_aos, gt_annos, dt_annos = run_reference(E, KC, ids, labels, results, c["classes"])
        p = f"{name}/"
        out.update({p + "ids": ids, p + "label_text": np.array(labels), p + "result_text": np.array(results),
                    p + "classes": np.array(c["classes"], dtype=np.int64), p + "texts": np.array(texts),
                    p + "min_overlaps": min_overlaps, p + "compute_aos": np.bool_(compute_aos)})
        for m, metric in enumerate(("bbox", "bev", "3d")):
            out[p + f"{metric}_precision"] = curves[m]["precision"]
            out[p + f"{metric}_thresholds"] = curves[m]["thresholds"]
        out[p + "bbox_orientation"] = curves[0]["orientation"]
        per_image = [mk.bev_3d_overlaps(E, g, d) for g, d in zip(gt_annos, dt_annos)]
        out[p + "margin"] = np.float64(mk.margin_of(per_image))
        ng = sum(len(a["name"]) for a in gt_annos)
        nd = sum(len(a["name"]) for a in dt_annos)
        print(f"{name}: {len(ids)} images, {ng} gt, {nd} dt, margin {float(out[p + 'margin']):.3g}")
        print(texts[0])
    np.savez_compressed(os.path.join(HERE, "kitti_coco.npz"), **out)


if __name__ == "__main__":
    main()
