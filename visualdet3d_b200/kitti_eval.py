"""KITTI object evaluation (2-D bbox / BEV / 3-D AP and AOS) on the GPU: the reference's `evaluate`, `get_official_eval_result` and
`get_coco_eval_result` (R/evaluator/kitti/evaluate.py, eval.py, kitti_common.py; R/ = visualDet3D in the reference tree), same inputs,
same strings, and its command line (R/evaluator/__main__.py):

    python -m visualdet3d_b200.kitti_eval --label_path L --result_path R --label_split_file val.txt --current_classes 0,1,2 [--coco]

Host code parses the label / result files and formats the text; everything from the overlaps to the precision curves is
`vd3d_kitti_eval` (csrc/kitti_eval.cu), which works per image and so accepts any number of images (the reference's 50-image
parts break below 50).  It runs on torch's current stream of the current CUDA device: no second CUDA context, no CPU fallback.
"""
from __future__ import annotations

import argparse
import io
import os
import pathlib
import re
import sys
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .loss_common import workspace

# eval.py:35-38 / 730-739: CLASS_NAMES of clean_data (index 5 is 'car' again) and class_to_name of the printed header
CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting', 5: 'car', 6: 'tractor', 7: 'trailer'}
NAME_TO_CLASS = {v: n for n, v in CLASS_TO_NAME.items()}
_LOWER_CODE = {'car': 0, 'pedestrian': 1, 'cyclist': 2, 'van': 3, 'person_sitting': 4, 'tractor': 6, 'trailer': 7}
_DONTCARE = -2
N_SAMPLE_PTS = 41
METRICS = ("bbox", "bev", "3d")

# eval.py:723-729: [moderate, easy] x [bbox, bev, 3d] x class
_OVERLAP_MOD = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7],
                         [0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7],
                         [0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7]])
_OVERLAP_EASY = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5, 0.5, 0.5],
                          [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5],
                          [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5]])
MIN_OVERLAPS = np.stack([_OVERLAP_MOD, _OVERLAP_EASY], axis=0)
# eval.py:818-827 (the second class_to_range of get_coco_eval_result): [first, last, number of] min overlaps per class
CLASS_TO_RANGE = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10], 3: [0.5, 0.95, 10], 4: [0.25, 0.7, 10],
                  5: [0.5, 0.95, 10], 6: [0.5, 0.95, 10], 7: [0.5, 0.95, 10]}


# ---- parsing (kitti_common.py:293-346) ------------------------------------------------------------------------------------
def get_label_anno(label_path) -> Dict[str, np.ndarray]:
    with open(label_path, 'r') as f:
        lines = f.readlines()
    content = [line.strip().split(' ') for line in lines]
    anno = {
        'name': np.array([x[0] for x in content]),
        'truncated': np.array([float(x[1]) for x in content]),
        'occluded': np.array([int(x[2]) for x in content]),
        'alpha': np.array([float(x[3]) for x in content]),
        'bbox': np.array([[float(v) for v in x[4:8]] for x in content]).reshape(-1, 4),
        # hwl in the file, lhw (camera) in the anno
        'dimensions': np.array([[float(v) for v in x[8:11]] for x in content]).reshape(-1, 3)[:, [2, 0, 1]],
        'location': np.array([[float(v) for v in x[11:14]] for x in content]).reshape(-1, 3),
        'rotation_y': np.array([float(x[14]) for x in content]).reshape(-1),
    }
    if len(content) != 0 and len(content[0]) == 16:
        anno['score'] = np.array([float(x[15]) for x in content])
    else:
        anno['score'] = np.zeros([len(anno['bbox'])])
    return anno


def get_label_annos(label_folder, image_ids=None) -> List[Dict[str, np.ndarray]]:
    """One anno dict per `{id:06d}.txt`; with image_ids None, every file named like that in the folder, by id."""
    if image_ids is None:
        prog = re.compile(r'^\d{6}.txt$')
        image_ids = sorted(int(p.stem) for p in pathlib.Path(label_folder).glob('*.txt') if prog.match(p.name))
    if not isinstance(image_ids, list):
        image_ids = list(range(image_ids))
    folder = pathlib.Path(label_folder)
    return [get_label_anno(folder / f"{idx:06d}.txt") for idx in image_ids]


# ---- device evaluation ------------------------------------------------------------------------------------------------------
def _class_codes(names: np.ndarray) -> np.ndarray:
    return np.array([_DONTCARE if n == "DontCare" else _LOWER_CODE.get(str(n).lower(), -1) for n in names], dtype=np.float64)


def _pack(annos, with_score: bool) -> np.ndarray:
    rows = []
    for a in annos:
        n = len(a['name'])
        cols = [a['bbox'].reshape(n, 4), a['alpha'].reshape(n, 1), a['dimensions'].reshape(n, 3), a['location'].reshape(n, 3),
                a['rotation_y'].reshape(n, 1), a['truncated'].reshape(n, 1), a['occluded'].reshape(n, 1), _class_codes(a['name'])[:, None]]
        if with_score:
            cols.append(a['score'].reshape(n, 1))
        rows.append(np.concatenate([c.astype(np.float64) for c in cols], 1))
    return np.ascontiguousarray(np.concatenate(rows, 0)) if rows else np.zeros((0, 16 if with_score else 15))


def _offsets(counts: np.ndarray) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)


class DeviceEval:
    """One evaluation staged on the current CUDA device: the constructor packs and uploads the annos, `run` launches the
    evaluator on the current stream (asynchronous), `collect` synchronises and returns the curves.  do_eval_v3 is the three in a row."""

    def __init__(self, gt_annos, dt_annos, current_classes: Sequence[int], min_overlaps: np.ndarray, compute_aos: bool):
        if len(gt_annos) != len(dt_annos):
            raise ValueError(f"{len(gt_annos)} ground-truth annos but {len(dt_annos)} result annos")
        n_img, n_cls = len(gt_annos), len(current_classes)
        if n_img == 0 or n_cls == 0:
            raise ValueError("nothing to evaluate: no images or no classes")
        classes = np.asarray(current_classes, dtype=np.int32)
        if classes.min() < 0 or classes.max() >= len(CLASS_TO_NAME):
            raise ValueError(f"class indices must be in 0..{len(CLASS_TO_NAME) - 1}: {current_classes}")
        mo = np.ascontiguousarray(np.asarray(min_overlaps, dtype=np.float64).reshape(-1, 3, n_cls))
        if mo.shape[0] == 0:
            raise ValueError("min_overlaps has no rows")
        self.ng = np.array([len(a['name']) for a in gt_annos], dtype=np.int64)
        self.nd = np.array([len(a['name']) for a in dt_annos], dtype=np.int64)
        self.offs = np.stack([_offsets(self.ng), _offsets(self.nd), _offsets(self.ng * self.nd), _offsets((self.nd + 31) // 32)])
        self.sizes = (n_img,) + tuple(int(x) for x in self.offs[:, -1])          # n_img, n_gt, n_dt, n_pairs, n_words
        self.n_cls, self.n_mo, self.compute_aos = n_cls, mo.shape[0], bool(compute_aos)
        self.dev = dev = torch.device("cuda", torch.cuda.current_device())
        self.ws, self.ws_bytes = workspace("vd3d_kitti_eval_workspace_bytes", n_img, self.sizes[1], self.sizes[2], self.sizes[4], n_cls,
                                           self.n_mo, device=dev)
        self.gt = torch.from_numpy(_pack(gt_annos, False)).to(dev)
        self.dt = torch.from_numpy(_pack(dt_annos, True)).to(dev)
        self.offs_d = torch.from_numpy(self.offs).to(dev)
        self.cls_d = torch.from_numpy(classes).to(dev)
        self.mo_d = torch.from_numpy(mo).to(dev)
        n_cfg = 9 * self.n_mo * n_cls
        f64 = dict(dtype=torch.float64, device=dev)
        self.overlaps = torch.empty(3 * self.sizes[3], **f64)
        self.precision = torch.empty(n_cfg * N_SAMPLE_PTS, **f64)
        self.orientation = torch.zeros(n_cfg // 3 * N_SAMPLE_PTS, **f64)
        self.thresholds = torch.empty(n_cfg * N_SAMPLE_PTS, **f64)
        self.n_thresh = torch.empty(n_cfg, dtype=torch.int32, device=dev)

    def run(self) -> "DeviceEval":
        n_img, n_gt, n_dt, n_pairs, n_words = self.sizes
        _lib.call("vd3d_kitti_eval", self.gt.data_ptr(), self.dt.data_ptr(), self.offs_d.data_ptr(), n_img, n_gt, n_dt, n_pairs, n_words,
                  self.cls_d.data_ptr(), self.n_cls, self.mo_d.data_ptr(), self.n_mo, int(self.compute_aos), self.overlaps.data_ptr(),
                  self.precision.data_ptr(), self.orientation.data_ptr(), self.thresholds.data_ptr(), self.n_thresh.data_ptr(),
                  self.ws.data_ptr(), self.ws_bytes, torch.cuda.current_stream(self.dev).cuda_stream)
        return self

    def collect(self, return_overlaps: bool = False) -> Dict[str, Dict[str, np.ndarray]]:
        n_thresh = self.n_thresh.cpu().numpy()
        if n_thresh.max() > N_SAMPLE_PTS:   # the reference fails on the same input (eval.py:547 writes past 41 entries)
            raise ValueError(f"a configuration selected {int(n_thresh.max())} recall thresholds, more than {N_SAMPLE_PTS}")
        shape = (3, self.n_cls, 3, self.n_mo, N_SAMPLE_PTS)
        precision = self.precision.cpu().numpy().reshape(shape)
        thresholds = self.thresholds.cpu().numpy().reshape(shape)
        orientation = self.orientation.cpu().numpy().reshape(shape[1:])
        out = {}
        for m, name in enumerate(METRICS):
            out[name] = {"precision": precision[m], "thresholds": thresholds[m],
                         "orientation": orientation if m == 0 else np.zeros_like(orientation)}
        if return_overlaps:
            ov, o = self.overlaps.cpu().numpy().reshape(3, -1), self.offs[2]
            out["overlaps"] = [ov[:, o[i]:o[i + 1]].reshape(3, self.nd[i], self.ng[i]) for i in range(self.sizes[0])]
        return out


def do_eval_v3(gt_annos, dt_annos, current_classes: Sequence[int], min_overlaps: np.ndarray, compute_aos: bool,
               return_overlaps: bool = False) -> Dict[str, Dict[str, np.ndarray]]:
    """eval.py do_eval_v3 with difficulties (0, 1, 2): per metric, `precision` / `orientation` / `thresholds`
    [class][difficulty][row][41] as eval_class returns them (orientation is computed for bbox only, the one printed).
    min_overlaps [rows][3][len(current_classes)], any number of rows, all evaluated in one device call.  return_overlaps adds
    "overlaps": per image a [3][dt][gt] float64 array."""
    return DeviceEval(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos).run().collect(return_overlaps)


def rotate_iou(boxes: torch.Tensor, query_boxes: torch.Tensor, criterion: int = -1) -> torch.Tensor:
    """rotate_iou_gpu_eval on device tensors: boxes [N][5], query_boxes [K][5] (x, y, dx, dy, angle) -> [N][K] float32."""
    b = boxes.to(torch.float32).contiguous()
    q = query_boxes.to(device=b.device, dtype=torch.float32).contiguous()
    if b.dim() != 2 or b.shape[1] != 5 or q.dim() != 2 or q.shape[1] != 5:
        raise ValueError("rotate_iou: boxes and query_boxes must be [n][5]")
    out = torch.zeros(b.shape[0], q.shape[0], dtype=torch.float32, device=b.device)
    _lib.call("vd3d_kitti_rotate_iou", b.data_ptr(), b.shape[0], q.data_ptr(), q.shape[0], int(criterion), out.data_ptr(),
              torch.cuda.current_stream(b.device).cuda_stream)
    return out


# ---- text (eval.py:597-601, 705-790) ------------------------------------------------------------------------------------------
def get_mAP_v2(prec: np.ndarray) -> np.ndarray:
    sums = 0
    for i in range(1, prec.shape[-1]):
        sums = sums + prec[..., i]
    return sums / 40 * 100


def _maps(metrics, compute_aos: bool):
    """do_eval_v2's (mAP_bbox, mAP_bev, mAP_3d, mAP_aos) [class][difficulty][row] from do_eval_v3's curves; mAP_aos is None without AOS."""
    bbox, bev, d3 = (get_mAP_v2(metrics[m]["precision"]) for m in METRICS)
    return bbox, bev, d3, get_mAP_v2(metrics["bbox"]["orientation"]) if compute_aos else None


def do_eval_v2(gt_annos, dt_annos, current_classes: Sequence[int], min_overlaps: np.ndarray, compute_aos: bool = False):
    """eval.py do_eval_v2 with difficulties (0, 1, 2): mAP_bbox, mAP_bev, mAP_3d [class][difficulty][row] and mAP_aos (None unless
    compute_aos; bbox only).  The reference runs eval_class once per metric; here the three metrics are one device call."""
    return _maps(do_eval_v3(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos), compute_aos)


def coco_min_overlaps(overlap_ranges: np.ndarray) -> np.ndarray:
    """do_coco_style_eval's [10][metric][class] min overlaps from overlap_ranges [first, last, number][metric][class]."""
    min_overlaps = np.zeros([10, *overlap_ranges.shape[1:]])
    for i in range(overlap_ranges.shape[1]):
        for j in range(overlap_ranges.shape[2]):
            start, stop, num = overlap_ranges[:, i, j]
            min_overlaps[:, i, j] = np.linspace(start, stop, int(num))
    return min_overlaps


def _row_mean(maps):
    return tuple(None if m is None else m.mean(-1) for m in maps)


def do_coco_style_eval(gt_annos, dt_annos, current_classes: Sequence[int], overlap_ranges: np.ndarray, compute_aos: bool):
    """eval.py do_coco_style_eval: do_eval_v2 over ten min-overlap rows spread from overlap_ranges [first, last, number][metric][class]
    (see get_coco_eval_result for the integer `number`), each mAP meaned over the rows: [class][difficulty], mAP_aos None without AOS."""
    return _row_mean(do_eval_v2(gt_annos, dt_annos, current_classes, coco_min_overlaps(overlap_ranges), compute_aos))


def _coco_overlap_ranges(classes: Sequence[int]) -> np.ndarray:
    overlap_ranges = np.zeros([3, 3, len(classes)])
    for i, curcls in enumerate(classes):
        overlap_ranges[:, :, i] = np.array(CLASS_TO_RANGE[curcls])[:, np.newaxis]
    return overlap_ranges


def _print_str(value) -> str:
    s = io.StringIO()
    print(value, file=s)
    return s.getvalue()


def _class_indices(current_classes) -> List[int]:
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    return [NAME_TO_CLASS[c] if isinstance(c, str) else c for c in current_classes]


def _compute_aos(dt_annos) -> bool:
    """AOS only when the first result anno with rows has a real alpha (the 2-D result writer puts -10 there)."""
    for anno in dt_annos:
        if anno['alpha'].shape[0] != 0:
            return bool(anno['alpha'][0] != -10)
    return False


def format_official_result(metrics, current_classes, compute_aos: bool) -> str:
    """The text get_official_eval_result prints, from do_eval_v3's precision / orientation arrays."""
    classes = _class_indices(current_classes)
    min_overlaps = MIN_OVERLAPS[:, :, classes]
    result = ''
    for j, curcls in enumerate(classes):
        for i in range(min_overlaps.shape[0]):
            ap = {m: ", ".join(f"{v:.2f}" for v in get_mAP_v2(metrics[m]["precision"][j, :, i])) for m in METRICS}
            result += _print_str((f"{CLASS_TO_NAME[curcls]} "
                                  "AP(Average Precision)@{:.2f}, {:.2f}, {:.2f}:".format(*min_overlaps[i, :, j])))
            result += _print_str(f"bbox AP:{ap['bbox']}")
            result += _print_str(f"bev  AP:{ap['bev']}")
            result += _print_str(f"3d   AP:{ap['3d']}")
            if compute_aos:
                aos = ", ".join(f"{v:.2f}" for v in get_mAP_v2(metrics["bbox"]["orientation"][j, :, i]))
                result += _print_str(f"aos  AP:{aos}")
    return result


def format_coco_result(metrics, current_classes, compute_aos: bool) -> str:
    """The text get_coco_eval_result prints, from do_eval_v3's precision / orientation arrays over the ten COCO rows."""
    classes = _class_indices(current_classes)
    mAPbbox, mAPbev, mAP3d, mAPaos = _row_mean(_maps(metrics, compute_aos))
    result = ''
    for j, curcls in enumerate(classes):
        o_range = np.array(CLASS_TO_RANGE[curcls])[[0, 2, 1]]
        o_range[1] = (o_range[2] - o_range[0]) / (o_range[1] - 1)
        result += _print_str((f"{CLASS_TO_NAME[curcls]} "
                              "coco AP@{:.2f}:{:.2f}:{:.2f}:".format(*o_range)))
        result += _print_str(f"bbox AP:{mAPbbox[j, 0]:.2f}, {mAPbbox[j, 1]:.2f}, {mAPbbox[j, 2]:.2f}")
        result += _print_str(f"bev  AP:{mAPbev[j, 0]:.2f}, {mAPbev[j, 1]:.2f}, {mAPbev[j, 2]:.2f}")
        result += _print_str(f"3d   AP:{mAP3d[j, 0]:.2f}, {mAP3d[j, 1]:.2f}, {mAP3d[j, 2]:.2f}")
        if compute_aos:
            result += _print_str(f"aos  AP:{mAPaos[j, 0]:.2f}, {mAPaos[j, 1]:.2f}, {mAPaos[j, 2]:.2f}")
    return result


def get_coco_eval_result(gt_annos, dt_annos, current_classes) -> str:
    """eval.py get_coco_eval_result (camera frame: z_axis 1, z_center 1.0): per class, AP averaged over ten min overlaps, 0.50 .. 0.95
    for Car / Van (and 'car', tractor, trailer), 0.25 .. 0.70 for Pedestrian / Person_sitting / Cyclist, for every metric; all three
    metrics and ten rows are one device call.

    One deliberate departure: the reference passes the number of rows to np.linspace as a float64 taken from its overlap_ranges array,
    which numpy >= 1.18 refuses with a TypeError, so the reference's function cannot run on any current numpy.  Here that number is cast
    to int, which gives the row values an older numpy computed.  The text is otherwise the reference's, character for character."""
    classes = _class_indices(current_classes)
    compute_aos = _compute_aos(dt_annos)
    metrics = do_eval_v3(gt_annos, dt_annos, classes, coco_min_overlaps(_coco_overlap_ranges(classes)), compute_aos)
    return format_coco_result(metrics, classes, compute_aos)


def get_official_eval_result(gt_annos, dt_annos, current_classes) -> str:
    """eval.py get_official_eval_result (difficulties 0, 1, 2; camera frame: z_axis 1, z_center 1.0)."""
    classes = _class_indices(current_classes)
    compute_aos = _compute_aos(dt_annos)
    metrics = do_eval_v3(gt_annos, dt_annos, classes, MIN_OVERLAPS[:, :, classes], compute_aos)
    return format_official_result(metrics, classes, compute_aos)


def _read_imageset_file(path) -> List[int]:
    with open(path, 'r') as f:
        return [int(line) for line in f.readlines()]


def _read_annos(label_path, result_path, label_split_file):
    """(gt_annos, dt_annos): result files (sorted by id) are paired with the split's ids by position."""
    dt_annos = get_label_annos(result_path)
    gt_annos = get_label_annos(label_path, _read_imageset_file(label_split_file))
    return gt_annos, dt_annos


def evaluate(label_path, result_path, label_split_file, current_classes=[0], gpu: Optional[int] = 0) -> List[str]:
    """evaluate.py evaluate: result files (sorted by id) are paired with the split's ids by position; one string per class."""
    with torch.cuda.device(gpu):
        gt_annos, dt_annos = _read_annos(label_path, result_path, label_split_file)
        return [get_official_eval_result(gt_annos, dt_annos, c) for c in current_classes]


# ---- command line (R/evaluator/__main__.py) ---------------------------------------------------------------------------------
def _parse_classes(text: str) -> List[int]:
    classes = []
    for tok in (t.strip() for t in text.split(",")):
        if tok.isdigit() and int(tok) in CLASS_TO_NAME:
            classes.append(int(tok))
        elif tok in NAME_TO_CLASS:
            classes.append(NAME_TO_CLASS[tok])
        else:
            raise ValueError(f"unknown class {tok!r}: use indices 0..{len(CLASS_TO_NAME) - 1} or the names "
                             + ", ".join(NAME_TO_CLASS))
    return classes


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m visualdet3d_b200.kitti_eval",
                                 description="The reference's KITTI object evaluator command line on the GPU: one official AP string "
                                             "per class, and with --coco the COCO-style AP string per class after them.")
    ap.add_argument("--evaluator", default="kitti_obj", help="kitti_obj (the only evaluator here)")
    ap.add_argument("--label_path", required=True, help="folder of KITTI label files {id:06d}.txt")
    ap.add_argument("--result_path", required=True, help="folder of result files {id:06d}.txt, paired with the split by sorted position")
    ap.add_argument("--label_split_file", default="val.txt", help="image ids to evaluate, one per line")
    ap.add_argument("--current_classes", default="0", help="comma-separated class indices or names, e.g. 0,1,2 or Car,Pedestrian")
    ap.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    ap.add_argument("--coco", action="store_true", help="also print the COCO-style AP (ten min overlaps per class)")
    args = ap.parse_args(argv)
    if args.evaluator.lower() == "kitti_depth":
        ap.error("the depth evaluator (kitti_depth) is out of scope for this package: only kitti_obj is available")
    if args.evaluator.lower() != "kitti_obj":
        ap.error(f"unknown evaluator {args.evaluator!r}: only kitti_obj is available (the depth evaluator is out of scope)")
    try:
        args.current_classes = _parse_classes(args.current_classes)
    except ValueError as e:
        ap.error(str(e))
    for flag, path, ok in (("--label_path", args.label_path, os.path.isdir), ("--result_path", args.result_path, os.path.isdir),
                           ("--label_split_file", args.label_split_file, os.path.isfile)):
        if not ok(path):
            ap.error(f"{flag} {path!r} does not exist")
    return args


def main(label_path, result_path, label_split_file, current_classes=[0], gpu: int = 0, coco: bool = False) -> None:
    """Print what evaluate() returns, one string per class; with coco, the COCO-style string per class after them (the same annos)."""
    with torch.cuda.device(gpu):
        gt_annos, dt_annos = _read_annos(label_path, result_path, label_split_file)
        for c in current_classes:
            print(get_official_eval_result(gt_annos, dt_annos, c))
        if coco:
            for c in current_classes:
                print(get_coco_eval_result(gt_annos, dt_annos, c))


if __name__ == "__main__":
    a = parse_args(sys.argv[1:])
    try:
        main(a.label_path, a.result_path, a.label_split_file, a.current_classes, a.gpu, a.coco)
    except (OSError, ValueError) as e:             # unreadable files, result / split count mismatch
        sys.exit(f"kitti_eval: {e}")
