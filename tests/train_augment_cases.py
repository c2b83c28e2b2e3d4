"""The five shipped `train_augmentation` lists (R/config/*_example) and the seeded frames / calibration / labels the training
augmentation is pinned on (tests/golden/make_golden_train_augment.py, tests/test_train_augment_*.py, tools/bench_train_augment.py)."""
import numpy as np

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def _e(name, **kw):
    return {"type_name": name, "keywords": kw} if kw else {"type_name": name}


def _chain1(size=(288, 1280), crop_top=100):
    return [_e("ConvertToFloat"),
            _e("PhotometricDistort", distort_prob=1.0, contrast_lower=0.5, contrast_upper=1.5, saturation_lower=0.5, saturation_upper=1.5,
               hue_delta=18.0, brightness_delta=32),
            _e("CropTop", crop_top_index=crop_top), _e("Resize", size=size), _e("RandomMirror", mirror_prob=0.5),
            _e("Normalize", mean=MEAN, stds=STD)]


def _shuffle():
    return _e("Shuffle", aug_list=[_e("RandomBrightness", distort_prob=1.0), _e("RandomContrast", distort_prob=1.0, lower=0.6, upper=1.4),
                                   _e("Compose", aug_list=[_e("ConvertColor", transform="HSV"),
                                                           _e("RandomSaturation", distort_prob=1.0, lower=0.6, upper=1.4),
                                                           _e("ConvertColor", current="HSV", transform="RGB")])])


def monoflex_list(size=(384, 1280)):
    return [_e("RandomWarpAffine", output_w=size[1], output_h=size[0]), _e("ConvertToFloat"), _shuffle(),
            _e("RandomMirror", mirror_prob=0.5), _e("FilterObject"), _e("Normalize", mean=MEAN, stds=STD)]


def km3d_list(size=(384, 1280)):
    return [_e("ConvertToFloat"), _e("RandomWarpAffine", output_w=size[1], output_h=size[0]), _shuffle(),
            _e("RandomEigenvalueNoise", alphastd=0.1), _e("RandomMirror", mirror_prob=0.5), _e("FilterObject"),
            _e("Normalize", mean=MEAN, stds=STD)]


# name -> (train_augmentation list, stereo dataset?)
LISTS = {"stereo3d": (_chain1(), True), "yolo3d": (_chain1(), False), "retinanet": (_chain1(), False),
         "monoflex": (monoflex_list(), False), "km3d": (km3d_list(), False)}
NAMES = list(LISTS)
SIZES = [(375, 1242), (370, 1224), (376, 1241)]

P2 = np.array([[7.215377e+02, 0.0, 6.095593e+02, 4.485728e+01], [0.0, 7.215377e+02, 1.728540e+02, 2.163791e-01], [0.0, 0.0, 1.0, 2.745884e-03]])
P3 = np.array([[7.215377e+02, 0.0, 6.095593e+02, -3.395242e+02], [0.0, 7.215377e+02, 1.728540e+02, 2.199936e+00], [0.0, 0.0, 1.0, 2.729905e-03]])


def frame(seed, H, W):
    """Smooth-ish uint8 content plus noise, so both the interpolation and the per-pixel colour programs see real variation."""
    rng = np.random.RandomState(seed)
    base = rng.randint(0, 256, (H // 8 + 2, W // 8 + 2, 3)).astype(np.float32)
    img = np.kron(base, np.ones((8, 8, 1), dtype=np.float32))[:H, :W] * 0.7 + rng.randint(0, 77, (H, W, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


LABEL_FIELDS = ("bbox_l", "bbox_t", "bbox_r", "bbox_b", "x", "ry", "alpha")


def labels(seed, H, W, make):
    """Six objects: four inside the frame, one near each side edge (dropped by FilterObject after some warps).  `make()` returns an
    object with KittiObj's attributes."""
    rng = np.random.RandomState(seed + 7)
    out = []
    for i in range(6):
        o = make()
        o.type = "Car"
        cx = [0.2, 0.4, 0.6, 0.8, 0.01, 0.99][i] * W
        cy = rng.uniform(0.45, 0.75) * H
        bw, bh = rng.uniform(30, 200), rng.uniform(20, 120)
        o.bbox_l, o.bbox_r = float(cx - bw / 2), float(cx + bw / 2)
        o.bbox_t, o.bbox_b = float(cy - bh / 2), float(cy + bh / 2)
        o.h, o.w, o.l = float(rng.uniform(1.4, 1.7)), float(rng.uniform(1.5, 1.9)), float(rng.uniform(3.5, 4.5))
        o.z = float(rng.uniform(5, 50))
        o.x = float((cx - P2[0, 2]) * o.z / P2[0, 0])
        o.y = float(rng.uniform(1.4, 1.8))
        o.ry = float(rng.uniform(-np.pi, np.pi))
        o.alpha = float(o.ry - np.arctan2(o.x, o.z))
        o.truncated, o.occluded = 0.0, 0
        out.append(o)
    return out


def label_array(objs):
    return np.array([[float(getattr(o, f)) for f in LABEL_FIELDS] for o in objs], dtype=np.float64).reshape(-1, len(LABEL_FIELDS))
