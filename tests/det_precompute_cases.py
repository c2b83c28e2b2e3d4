"""Constructed inputs for the anchor-prior accumulation (csrc/anchor_prior.cu) and the det_precompute CLI.

kernel_cases(): each case is one batch (anchors [N, 4] float32, a bin per anchor, B frames x T classes of boxes and (z, sin 2a, cos 2a)
rows, a threshold) and states the edge it reaches in `claim`; tests/test_det_precompute_cpu.py checks that it does.  The expected
accumulator states come from the reference's own calc_iou / torch.max and the script's loop (tests/golden/make_golden_det_precompute.py).

write_tree() / write_config(): a constructed KITTI tree (two frame sizes; Car / Pedestrian / Cyclist / DontCare rows; rows dropped by
occlusion and by min_z; frames with no kept label) and small configs holding the fields det_precompute reads, with the reference
examples' anchors and test lists (TEST_LISTS restates the six examples' lists).  `stereo3d_f64`'s Resize size is a numpy array, so its
labels become numpy float64 and the IoU float64; its `Van` class has no object in the split (the NaN w / h / l columns)."""
from __future__ import annotations

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _seg(boxes, gt3=None):
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 4)
    if gt3 is None:
        gt3 = np.stack([np.full(len(boxes), 10.0), np.full(len(boxes), 0.25), np.full(len(boxes), 0.5)], axis=1)
    return boxes, np.asarray(gt3, dtype=np.float64).reshape(-1, 3)


def _case(cid, claim, anchors, bins, n_bins, segs, T=1, thr=0.5, f64=False):
    """segs: B * T (boxes, gt3) pairs, frame-major."""
    off = np.zeros(len(segs) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(b) for b, _ in segs])
    boxes = np.concatenate([b for b, _ in segs]) if off[-1] else np.zeros((0, 4))
    gt3 = np.concatenate([g for _, g in segs]) if off[-1] else np.zeros((0, 3))
    return dict(id=cid, claim=claim, anchors=np.asarray(anchors, dtype=np.float32).reshape(-1, 4), bins=np.asarray(bins, dtype=np.int64),
                n_bins=n_bins, T=T, B=len(segs) // T, offsets=off, boxes=boxes.astype(np.float64 if f64 else np.float32), gt3=gt3,
                thr=thr, f64=f64)


def grid_table(H, W, ratios=(0.5, 1.0, 2.0), scales=(1.0, 2 ** 0.5, 2.0, 2 ** 1.5)):
    """A Stereo3D-style single-level table (stride 16, size 24) and its float32-form bins."""
    from visualdet3d_b200.anchor_prior import bin_table32
    from visualdet3d_b200.anchors import grid_anchors
    a32 = grid_anchors((H, W), [4], [16], [24], np.array(ratios), np.array(scales)).astype(np.float32)
    rows, cols = bin_table32(a32, [24], np.array(ratios), np.array(scales))
    return a32, rows * len(ratios) + cols, len(ratios) * len(scales)


def _random_frames(rng, a32, B, T, kmax, f64_scale=None):
    segs = []
    for _ in range(B * T):
        K = rng.randint(0, kmax + 1)
        picks = a32[rng.randint(0, len(a32), K)].astype(np.float64)
        jitter = rng.uniform(-4, 4, (K, 4))
        boxes = picks + jitter
        if f64_scale is not None:
            boxes = boxes * f64_scale
        z = rng.uniform(5, 60, K)
        alpha = rng.uniform(-np.pi, np.pi, K)
        segs.append(_seg(boxes, np.stack([z, np.sin(2 * alpha), np.cos(2 * alpha)], axis=1)))
    return segs


NEG_COPIES = 20000
ANCHOR_AREA32 = 16785408                  # float32(4097 * 4097)
AREA_BOX_H = 8392704.25 / 4097            # 4097 * h falls between half the float32 area and half the exact one


def negative_variance_z():
    """A z whose NEG_COPIES equal copies, summed in order, make the script's EX_2 - avg ** 2 round below zero (std NaN).  Fewer copies
    cannot: the + 1e-8 in the script's divisor keeps the exact difference above a few copies' rounding error."""
    e = NEG_COPIES + 1e-8
    for k in range(1, 4000):
        x = 1.0 + k / 7.0
        s = np.add.accumulate(np.full(NEG_COPIES, x))[-1]            # sequential, like the script's +=
        q = np.add.accumulate(np.full(NEG_COPIES, x ** 2))[-1]
        if q / e - (s / e) ** 2 < 0:
            return x
    raise AssertionError("no z found")


def kernel_cases():
    cases = []
    sq = [[0, 0, 10, 10]]
    cases.append(_case("iou_exactly_half", "anchor 0's IoU is exactly 0.5 and not positive; anchor 1 (IoU 1) is",
                       [[0, 0, 10, 10], [0, 0, 20, 10]], [0, 1], 2, [_seg([[0, 0, 20, 10]])]))
    cases.append(_case("identical_gts", "two identical boxes: the argmax takes the first, so the sums hold the first row",
                       sq, [0], 1, [_seg([[0, 0, 10, 10], [0, 0, 10, 10]], [[7.0, 0.1, 0.2], [9.0, 0.3, 0.4]])]))
    cases.append(_case("tied_gts", "the anchor's IoU ties (0.5) between two different boxes: the first wins",
                       sq, [0], 1, [_seg([[0, 0, 10, 20], [0, -10, 10, 10]], [[3.0, 0.5, 0.5], [4.0, 0.6, 0.6]])], thr=0.4))
    cases.append(_case("zero_area_gt", "a zero-area box has IoU 0 everywhere: not usable, never an argmax over a real box",
                       [[0, 0, 10, 10], [5, 5, 15, 15]], [0, 1], 2, [_seg([[5, 5, 5, 5], [0, 0, 10, 10]])]))
    cases.append(_case("unreachable_gt", "a box no anchor overlaps is not usable",
                       [[0, 0, 10, 10], [5, 5, 15, 15]], [0, 1], 2, [_seg([[100, 100, 120, 130], [0, 0, 10, 10]])]))
    cases.append(_case("threshold_f32", "IoU 0.6f: positive against 0.6 in float64 but not in float32 (the comparison's dtype)",
                       [[0, 0, 10, 10]], [0], 1, [_seg([[0, 0, 10, 6.0]])], thr=0.6))
    cases.append(_case("threshold_f64", "the float64 IoU of the same pair is 0.6 exactly, not > 0.6",
                       [[0, 0, 10, 10]], [0], 1, [_seg([[0, 0, 10, 6.0]])], thr=0.6, f64=True))
    cases.append(_case("f64_threshold_flip", "float64 box [0, 0, 10, 6.0000001]: its float64 IoU is > 0.6 (positive, usable); "
                       "rounded to float32 it is 0.6f, not > 0.6f", [[0, 0, 10, 10]], [0], 1, [_seg([[0, 0, 10, 6.0000001]])], thr=0.6,
                       f64=True))
    cases.append(_case("f64_threshold_flip_as_f32", "the same box as float32 values: no positive, not usable", [[0, 0, 10, 10]], [0], 1,
                       [_seg([[0, 0, 10, 6.0000001]])], thr=0.6))
    cases.append(_case("f64_anchor_area_f32", f"anchor [0, 0, 4097, 4097], whose area rounds to {ANCHOR_AREA32} in float32 "
                       f"(exactly {4097 * 4097}): the box's IoU is > 0.5 only with the float32-rounded area; a float64 area, or float32 "
                       "throughout, puts it at or below 0.5", [[0, 0, 4097, 4097]], [0], 1, [_seg([[0, 0, 4097, AREA_BOX_H]])], f64=True))
    few = [_seg(sq) for _ in range(9)]
    cases.append(_case("few_positives", "bin 0 receives 9 positives (< 10: the -100 / 1e10 sentinel)", sq, [0], 1, few))
    same = [_seg(sq, [[12.5, 0.0, 1.0]]) for _ in range(12)]
    cases.append(_case("same_z", "12 positives with one (z, sin, cos): std < 1e-3, the sentinel", sq, [0], 1, same))
    x = negative_variance_z()
    cases.append(_case("negative_variance", f"{NEG_COPIES} positives of one z in one bin: EX_2 - avg ** 2 rounds negative, std NaN, "
                       "the sentinel", sq * NEG_COPIES, [0] * NEG_COPIES, 1, [_seg(sq, [[x, 0.5, 0.5]])]))
    rng = np.random.RandomState(5)
    big = rng.uniform(0, 200, (512, 2))
    full = _seg(np.concatenate([big, big + rng.uniform(5, 40, (512, 2))], axis=1))
    a32, bins, nb = grid_table(96, 320)
    cases.append(_case("k_edges", "segments with K = 0 and K = 512 (the largest the entry accepts)", a32, bins, nb,
                       [_seg(np.zeros((0, 4))), full, _seg(np.zeros((0, 4))), _seg(a32[:3].astype(np.float64))], T=2))
    cases.append(_case("many_frames_f32", "1440 anchors (6 IoU blocks, the last partial), 120 per bin x 20 frames x 2 classes: the walk "
                       "crosses its 1024-pair step", a32, bins, nb, _random_frames(rng, a32, 20, 2, 6), T=2))
    cases.append(_case("many_frames_f64", "the same in float64 boxes (Resize's numpy scale factor)", a32, bins, nb,
                       _random_frames(rng, a32, 20, 2, 6, f64_scale=288 / 275), T=2, f64=True))
    return cases


def label(typ, box, z=20.0, alpha=0.3):
    """A label row with the fields the accumulator reads."""
    import types
    return types.SimpleNamespace(type=typ, bbox_l=box[0], bbox_t=box[1], bbox_r=box[2], bbox_b=box[3], z=z, alpha=alpha)


# one 16x16 cell: anchor 0 is [3, 3, 13, 13]; the box's IoU with it is 0.6 + 1e-8 in float64 and 0.6f in float32
FLIP_CFG = dict(pyramid_levels=[4], strides=[16], sizes=[10], ratios=np.array([1.0]), scales=np.array([1.0, 2.0]))
FLIP_BOX = (3.0, 3.0, 13.0, 9.0000001)


def dtype_frames():
    f64 = tuple(np.float64(v) for v in FLIP_BOX)
    return [[label("Car", f64), label("Pedestrian", FLIP_BOX)],          # one frame, two dtypes
            [label("Car", FLIP_BOX), label("Pedestrian", f64)],          # each class changes dtype
            [label("Car", f64)]]



# ---- the constructed KITTI tree ------------------------------------------------------------------------------------------------------

SIZES = [(375, 1242), (370, 1224)]
N_FRAMES = 40


def _label_rows(rng, i, H, W):
    rows = []
    if i % 9 == 4:                                          # frames with no kept label: only rows the filters drop
        return [("DontCare", 0, 0.0, 10.0), ("Car", 3, 1.0, 20.0), ("Pedestrian", 0, 0.2, 1.5)]
    n = rng.randint(3, 9)
    for k in range(n):
        typ = ["Car", "Car", "Car", "Pedestrian", "Cyclist", "DontCare"][rng.randint(0, 6)]
        occ = 3 if rng.rand() < 0.1 else rng.randint(0, 2)
        z = 2.0 if rng.rand() < 0.08 else rng.uniform(4, 60)
        rows.append((typ, occ, rng.uniform(-np.pi, np.pi), z))
    return rows


def write_tree(tmp: str, n_frames: int = N_FRAMES):
    """KITTI training / testing trees under tmp/kitti and the train / val split files; returns (raw training dir, split dir)."""
    import cv2
    import train_augment_cases as tac
    rng = np.random.RandomState(11)
    split = os.path.join(tmp, "split")
    os.makedirs(split, exist_ok=True)
    for part in ("training", "testing"):
        raw = os.path.join(tmp, "kitti", part)
        for d in ("calib", "image_2", "label_2"):
            os.makedirs(os.path.join(raw, d), exist_ok=True)
    fmt = lambda a: " ".join("%.12e" % v for v in np.asarray(a).reshape(-1))
    for part, count in (("training", n_frames), ("testing", 3)):
        raw = os.path.join(tmp, "kitti", part)
        for i in range(count):
            H, W = SIZES[(i // 3) % 2]
            idx = "%06d" % i
            cv2.imwrite(os.path.join(raw, "image_2", idx + ".png"), tac.frame(i % 7, H, W))
            P2 = tac.P2.copy()
            P2[0, 0] += i * 0.5
            with open(os.path.join(raw, "calib", idx + ".txt"), "w") as f:
                f.write(f"P0: {fmt(P2)}\nP1: {fmt(P2)}\nP2: {fmt(P2)}\nP3: {fmt(tac.P3)}\n"
                        f"R0_rect: {fmt(np.eye(3))}\nTr_velo_to_cam: {fmt(np.eye(3, 4))}\nTr_imu_to_velo: {fmt(np.eye(3, 4))}\n")
            with open(os.path.join(raw, "label_2", idx + ".txt"), "w") as f:
                for typ, occ, alpha, z in _label_rows(rng, i, H, W):
                    h = rng.uniform(1.4, 1.9) if typ != "Pedestrian" else rng.uniform(1.5, 1.9)
                    w, l = rng.uniform(0.5, 2.0), rng.uniform(0.6, 4.5)
                    x = rng.uniform(-15, 15)
                    y = rng.uniform(1.0, 2.0)
                    u = P2[0, 0] * x / z + P2[0, 2]
                    v = P2[1, 1] * y / z + P2[1, 2]
                    bw, bh = P2[0, 0] * max(w, l) / z, P2[1, 1] * h / z
                    l_, t_ = np.clip(u - bw / 2, 0, W - 1), np.clip(v - bh, 0, H - 1)
                    r_, b_ = np.clip(u + bw / 2, 0, W - 1), np.clip(v, 0, H - 1)
                    f.write(f"{typ} 0.00 {occ} {alpha:.6f} {l_:.2f} {t_:.2f} {r_:.2f} {b_:.2f} {h:.2f} {w:.2f} {l:.2f} "
                            f"{x:.2f} {y:.2f} {z:.2f} {rng.uniform(-3, 3):.2f}\n")
    names = ["%06d" % i for i in range(n_frames)]
    with open(os.path.join(split, "train.txt"), "w") as f:
        f.write("".join(n + "\n" for n in names[: n_frames * 3 // 4]))
    with open(os.path.join(split, "val.txt"), "w") as f:
        f.write("".join(n + "\n" for n in names[n_frames * 3 // 4:]))
    return os.path.join(tmp, "kitti", "training"), split


_NORM = "edict(type_name='Normalize', keywords=edict(mean=np.array([0.485, 0.456, 0.406]), stds=np.array([0.229, 0.224, 0.225])))"
_F = "edict(type_name='ConvertToFloat')"
_CROP = "edict(type_name='CropTop', keywords=edict(crop_top_index=100))"
# the test lists of the reference's six example configs, restated
TEST_LISTS = {
    "Stereo3D": f"[{_F}, {_CROP}, edict(type_name='Resize', keywords=edict(size=(288, 1280))), {_NORM}]",
    "Yolo3D": f"[{_F}, {_CROP}, edict(type_name='Resize', keywords=edict(size=(288, 1280))), {_NORM}]",
    "RetinaNet": f"[{_F}, {_CROP}, edict(type_name='Resize', keywords=edict(size=(288, 1280))), {_NORM}]",
    "KM3D": f"[{_F}, edict(type_name='Resize', keywords=edict(size=(384, 1280))), {_NORM}]",
    "MonoFlex": f"[{_F}, edict(type_name='Resize', keywords=edict(size=(384, 1280))), {_NORM}]",
    "MonoDepth": f"[{_F}, edict(type_name='CropTop', keywords=edict(output_height=352)), "
                 f"edict(type_name='CropRight', keywords=edict(output_width=1216)), {_NORM}]",
}
_ANCHORS = "edict(pyramid_levels=[4], strides=[2 ** 4], sizes=[24], ratios=np.array({ratios}), scales=np.array([2 ** (i / 4.0) for i in range(16)]))"
# name: (obj_types, anchor ratios or None for anchor_prior = False, test list, max_occlusion, min_z)
CONFIGS = {
    "stereo3d": (["Car", "Pedestrian"], [0.5, 1, 2.0], TEST_LISTS["Stereo3D"], 2, 3),
    "stereo3d_f64": (["Car", "Pedestrian", "Van"], [0.5, 1, 2.0],
                     f"[{_F}, {_CROP}, edict(type_name='Resize', keywords=edict(size=np.array([288, 1280]))), {_NORM}]", 2, 3),
    "yolo3d": (["Car"], [0.5, 1], TEST_LISTS["Yolo3D"], 2, 3),
    "croptop": (["Car", "Pedestrian", "Cyclist"], [0.5, 1, 2.0], f"[{_F}, {_CROP}, {_NORM}]", 2, 3),
    "km3d": (["Car", "Pedestrian", "Cyclist"], None, TEST_LISTS["KM3D"], 4, 3),
}


def write_config(name: str, tmp: str, train_raw: str, split: str) -> str:
    """A config file with the fields det_precompute reads, for CONFIGS[name] and the tree written by write_tree."""
    types, ratios, test_list, max_occ, min_z = CONFIGS[name]
    pre = os.path.join(tmp, "pre", name)
    head = "edict()" if ratios is None else \
        f"edict(anchors_cfg={_ANCHORS.format(ratios=ratios)}, loss_cfg=edict(fg_iou_threshold=0.5))"
    src = f"""import numpy as np
from easydict import EasyDict as edict
cfg = edict()
cfg.obj_types = {types!r}
cfg.anchor_prior = {ratios is not None}
cfg.trainer = edict(gpu=0)
cfg.path = edict(data_path={train_raw!r}, test_path={os.path.join(os.path.dirname(train_raw), 'testing')!r}, preprocessed_path={pre!r})
cfg.data = edict(train_split_file={os.path.join(split, 'train.txt')!r}, val_split_file={os.path.join(split, 'val.txt')!r},
                 max_occlusion={max_occ}, min_z={min_z})
cfg.data.test_augmentation = {test_list}
cfg.detector = edict(name={name!r}, head={head})
"""
    os.makedirs(os.path.join(tmp, "configs"), exist_ok=True)
    path = os.path.join(tmp, "configs", name + ".py")
    with open(path, "w") as f:
        f.write(src)
    return path
