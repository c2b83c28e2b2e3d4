"""KITTI object evaluation (2-D bbox / BEV / 3-D AP and AOS) on the GPU: the reference's `evaluate`
(R/evaluator/kitti/evaluate.py, eval.py, kitti_common.py; R/ = visualDet3D in the reference tree), same inputs, same strings.

Host code parses the label / result files and formats the text; everything from the overlaps to the precision curves is
`vd3d_kitti_eval` (csrc/kitti_eval.cu), which works per image and so accepts any number of images (the reference's 50-image
parts break below 50).  It runs on torch's current stream of the current CUDA device: no second CUDA context, no CPU fallback.
"""
from __future__ import annotations

import io
import pathlib
import re
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
        mo = np.ascontiguousarray(np.asarray(min_overlaps, dtype=np.float64).reshape(2, 3, n_cls))
        self.ng = np.array([len(a['name']) for a in gt_annos], dtype=np.int64)
        self.nd = np.array([len(a['name']) for a in dt_annos], dtype=np.int64)
        self.offs = np.stack([_offsets(self.ng), _offsets(self.nd), _offsets(self.ng * self.nd), _offsets((self.nd + 31) // 32)])
        self.sizes = (n_img,) + tuple(int(x) for x in self.offs[:, -1])          # n_img, n_gt, n_dt, n_pairs, n_words
        self.n_cls, self.compute_aos = n_cls, bool(compute_aos)
        self.dev = dev = torch.device("cuda", torch.cuda.current_device())
        self.ws, self.ws_bytes = workspace("vd3d_kitti_eval_workspace_bytes", n_img, self.sizes[1], self.sizes[2], self.sizes[4], n_cls,
                                           device=dev)
        self.gt = torch.from_numpy(_pack(gt_annos, False)).to(dev)
        self.dt = torch.from_numpy(_pack(dt_annos, True)).to(dev)
        self.offs_d = torch.from_numpy(self.offs).to(dev)
        self.cls_d = torch.from_numpy(classes).to(dev)
        self.mo_d = torch.from_numpy(mo).to(dev)
        n_cfg = 18 * n_cls
        f64 = dict(dtype=torch.float64, device=dev)
        self.overlaps = torch.empty(3 * self.sizes[3], **f64)
        self.precision = torch.empty(n_cfg * N_SAMPLE_PTS, **f64)
        self.orientation = torch.zeros(n_cls * 6 * N_SAMPLE_PTS, **f64)
        self.thresholds = torch.empty(n_cfg * N_SAMPLE_PTS, **f64)
        self.n_thresh = torch.empty(n_cfg, dtype=torch.int32, device=dev)

    def run(self) -> "DeviceEval":
        n_img, n_gt, n_dt, n_pairs, n_words = self.sizes
        _lib.call("vd3d_kitti_eval", self.gt.data_ptr(), self.dt.data_ptr(), self.offs_d.data_ptr(), n_img, n_gt, n_dt, n_pairs, n_words,
                  self.cls_d.data_ptr(), self.n_cls, self.mo_d.data_ptr(), int(self.compute_aos), self.overlaps.data_ptr(),
                  self.precision.data_ptr(), self.orientation.data_ptr(), self.thresholds.data_ptr(), self.n_thresh.data_ptr(),
                  self.ws.data_ptr(), self.ws_bytes, torch.cuda.current_stream(self.dev).cuda_stream)
        return self

    def collect(self, return_overlaps: bool = False) -> Dict[str, Dict[str, np.ndarray]]:
        n_thresh = self.n_thresh.cpu().numpy()
        if n_thresh.max() > N_SAMPLE_PTS:   # the reference fails on the same input (eval.py:547 writes past 41 entries)
            raise ValueError(f"a configuration selected {int(n_thresh.max())} recall thresholds, more than {N_SAMPLE_PTS}")
        shape = (3, self.n_cls, 3, 2, N_SAMPLE_PTS)
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
    [class][difficulty][min_overlap][41] as eval_class returns them (orientation is computed for bbox only, the one printed).
    min_overlaps [2][3][len(current_classes)].  return_overlaps adds "overlaps": per image a [3][dt][gt] float64 array."""
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


def get_official_eval_result(gt_annos, dt_annos, current_classes) -> str:
    """eval.py get_official_eval_result (difficulties 0, 1, 2; camera frame: z_axis 1, z_center 1.0)."""
    classes = _class_indices(current_classes)
    compute_aos = _compute_aos(dt_annos)
    metrics = do_eval_v3(gt_annos, dt_annos, classes, MIN_OVERLAPS[:, :, classes], compute_aos)
    return format_official_result(metrics, classes, compute_aos)


def _read_imageset_file(path) -> List[int]:
    with open(path, 'r') as f:
        return [int(line) for line in f.readlines()]


def evaluate(label_path, result_path, label_split_file, current_classes=[0], gpu: Optional[int] = 0) -> List[str]:
    """evaluate.py evaluate: result files (sorted by id) are paired with the split's ids by position; one string per class."""
    with torch.cuda.device(gpu):
        dt_annos = get_label_annos(result_path)
        gt_annos = get_label_annos(label_path, _read_imageset_file(label_split_file))
        return [get_official_eval_result(gt_annos, dt_annos, c) for c in current_classes]
