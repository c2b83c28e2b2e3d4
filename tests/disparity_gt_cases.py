"""Constructed inputs for Stereo3D's disparity ground truth (visualdet3d_b200/csrc/disparity_gt.cu): grey stereo pairs for StereoBM,
LiDAR clouds, and a small KITTI tree for the precompute CLI.  Used by tests/golden/make_golden_disparity_gt.py (cv2 and the reference),
tests/test_disparity_gt_cpu.py and tests/test_disparity_gt_gpu.py.  Nothing here imports the package or the reference.

bm_cases(): dicts with id, left, right (uint8 [H, W]) and `claims`, the behaviours the case must reach (checked through the oracle's
cost volume by the CPU tests):
  "bands"     rows in bands at known disparities (`bands`: (row0, row1, d)); interior pixels choose d with a zero minimum cost
  "subpixel"  sub-pixel outputs of both signs
  "texture"   the texture filter (T < 10)
  "unique"    the uniqueness filter on a textured window
  "tie"       two adjacent cost indices share the minimum
  "saturate"  the prefilter reaches 0 and 62
  "defined"   at least one unfiltered output (the minimum legal shapes)
velo_cases(): dicts with id, points (float32 [N, 4]), the calibration (R0_rect, Tr_velo_to_cam 4x4, P2 3x4, baseline), H, W and
`margin` (True: every in-view point is at least MARGIN from a pixel boundary, a field-of-view edge and an integer 16 f b / z).
"""
import os

import numpy as np

ND = 192
MARGIN = 1e-6
MEAN = np.array([0.485, 0.456, 0.406])
STD = np.array([0.229, 0.224, 0.225])

# KITTI-like calibration (the shape of a raw KITTI calib file's values)
P2 = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]])
P3 = np.array([[721.5377, 0.0, 609.5593, -339.5242], [0.0, 721.5377, 172.854, 2.199936], [0.0, 0.0, 1.0, 0.002729905]])
R0 = np.eye(4)
R0[:3, :3] = [[0.9999239, 0.00983776, -0.007445048], [-0.009869795, 0.9999421, -0.004278459], [0.007402527, 0.004351614, 0.9999631]]
TR = np.eye(4)
TR[:3] = [[7.533745e-03, -9.999714e-01, -6.166020e-04, -4.069766e-03], [1.480249e-02, 7.280733e-04, -9.998902e-01, -7.631618e-02],
          [9.998621e-01, 7.523790e-03, 1.480755e-02, -2.717806e-01]]
BASELINE = 0.54


def _blur(a, sigma):
    import cv2
    return cv2.GaussianBlur(a, (0, 0), sigma)


def texture(seed, H, W, sigma=1.2):
    """Blurred noise stretched to 0..255, float64 [H, W]."""
    a = _blur(np.random.RandomState(seed).rand(H, W), sigma)
    return (a - a.min()) / (a.max() - a.min()) * 255


def shifted(tex, d):
    """left(x) = tex(x), right(x) = tex(x + d) for every row (d an integer or a float; linear interpolation), both uint8 [H, W]."""
    H, Wt = tex.shape
    W = Wt - ND - 2
    x = np.arange(W) + d
    x0 = np.floor(x).astype(int)
    f = x - x0
    right = tex[:, x0] * (1 - f) + tex[:, x0 + 1] * f
    return np.round(tex[:, :W]).astype(np.uint8), np.round(right).astype(np.uint8)


def banded(seed, H, W, bands, sigma=1.2):
    """Rows in bands (row0, row1, d): right = left shifted by d in each band."""
    tex = texture(seed, H, W + ND + 2, sigma)
    left = np.round(tex[:, :W]).astype(np.uint8)
    right = np.zeros_like(left)
    for r0, r1, d in bands:
        right[r0:r1] = shifted(tex[r0:r1], d)[1]
    return left, right


def _bands(H, ds):
    step = H // len(ds)
    return [(k * step, H if k == len(ds) - 1 else (k + 1) * step, d) for k, d in enumerate(ds)]


def bm_cases():
    cases = []
    b = _bands(200, [0, 1, 37, 190, 191])
    left, right = banded(1, 200, 480, b)
    cases.append(dict(id="bands_0_1_37_190_191", left=left, right=right, bands=b, claims=("bands",)))

    tex = texture(2, 96, 420 + ND + 2, sigma=2.5)
    l1, r1 = shifted(tex[:48], 20.3)
    l2, r2 = shifted(tex[48:], 57.7)
    cases.append(dict(id="fractional", left=np.concatenate([l1, l2]), right=np.concatenate([r1, r2]), claims=("subpixel",)))

    left, right = shifted(texture(3, 64, 400 + ND + 2, sigma=2.0), 30.5)
    cases.append(dict(id="half_pixel_tie", left=left, right=right, claims=("tie",)))

    tex = texture(4, 80, 420 + ND + 2)
    tex[20:60, 230:330] = 128.0                                    # flat patch, wider than the window
    left, right = shifted(tex, 12)
    cases.append(dict(id="flat_patch", left=left, right=right, claims=("texture",)))

    x = np.arange(420 + ND + 2)
    tex = np.tile(np.where(x % 8 < 4, 40.0, 200.0), (64, 1))         # period 8 < 25: equal minima 8 disparities apart
    left, right = shifted(tex, 9)
    cases.append(dict(id="stripes_period_8", left=left, right=right, claims=("unique",)))

    rng = np.random.RandomState(6)
    tex = np.zeros((72, 440 + ND + 2))
    for _ in range(60):
        y, xx, h, w = rng.randint(0, 60), rng.randint(0, 600), rng.randint(3, 20), rng.randint(3, 40)
        tex[y:y + h, xx:xx + w] = 255.0 if rng.rand() < 0.5 else 0.0
    tex += texture(7, 72, 440 + ND + 2, 1.0) * 0.02
    left, right = shifted(tex, 25)
    cases.append(dict(id="hard_edges", left=left, right=right, claims=("saturate",)))

    for seed, (H, W), ds in ((8, (288, 1280), [3, 24, 61, 120]), (9, (375, 1242), [7, 45, 88, 150, 180]), (10, (97, 451), [11, 60])):
        b = _bands(H, ds)
        left, right = banded(seed, H, W, b)
        cases.append(dict(id=f"shape_{H}x{W}", left=left, right=right, bands=b, claims=("bands",)))
    for seed, (H, W) in ((11, (26, 216)), (12, (26, 217))):
        left, right = banded(seed, H, W, [(0, H, 17)], sigma=1.0)
        cases.append(dict(id=f"min_{H}x{W}", left=left, right=right, claims=("defined",)))
    return cases


def interior(case):
    """(row0, row1, d): output rows whose whole window, with the prefilter's row above and below, lies inside one band."""
    return [(r0 + 13, r1 - 13, d) for r0, r1, d in case.get("bands", ()) if r1 - r0 > 26]


# ---- LiDAR --------------------------------------------------------------------------------------------------------------------------

def _M():
    return R0 @ TR


def project(points, P2_=P2, H=288, W=1280):
    """The device routine's float64 arithmetic: (u, v, cam z, in view)."""
    M = _M()
    p = points[:, :3].astype(np.float64)
    cam = [M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1] + M[r, 2] * p[:, 2] + M[r, 3] for r in range(3)]
    pix = [P2_[r, 0] * cam[0] + P2_[r, 1] * cam[1] + P2_[r, 2] * cam[2] + P2_[r, 3] for r in range(3)]
    u, v = pix[0] / (pix[2] + 1e-6), pix[1] / (pix[2] + 1e-6)
    ok = (u < W - 1) & (u >= 0) & (v < H - 1) & (v >= 0) & (p[:, 0] > 2)
    return u, v, cam[2], ok


def near_boundary(points, P2_=P2, H=288, W=1280, baseline=BASELINE, margin=MARGIN):
    """Per point: within `margin` of an integer u or v, a field-of-view edge, x = 2, or an integer 16 f b / z."""
    u, v, z, _ = project(points, P2_, H, W)
    disp = P2_[0, 0] * baseline / z * 16
    frac = lambda a: np.abs(a - np.round(a))
    return (frac(u) < margin) | (frac(v) < margin) | (np.abs(u - (W - 1)) < margin) | (np.abs(v - (H - 1)) < margin) | \
        (np.abs(points[:, 0].astype(np.float64) - 2) < margin) | (frac(disp) < margin)


def _from_pixels(u, v, z):
    """Velodyne points whose camera projection is (u, v) at camera depth z (float64 inverse of project)."""
    pix2 = z + P2[2, 3]
    rhs = np.stack([u * (pix2 + 1e-6) - P2[0, 2] * z - P2[0, 3], v * (pix2 + 1e-6) - P2[1, 2] * z - P2[1, 3]])
    cx = rhs[0] / P2[0, 0]
    cy = rhs[1] / P2[1, 1]
    cam = np.stack([cx, cy, z, np.ones_like(z)])
    return (np.linalg.inv(_M()) @ cam)[:3].T


def velo_cases():
    rng = np.random.RandomState(20)
    H, W = 288, 1280
    n = 40000
    u = rng.randint(0, W - 1, n) + rng.uniform(0.05, 0.95, n)
    v = rng.randint(0, H - 1, n) + rng.uniform(0.05, 0.95, n)
    z = rng.uniform(3.0, 70.0, n)
    pts = _from_pixels(u, v, z)
    # several points per pixel, in both depth orders: 2000 pixels get a near and a far point, near first for half of them
    k = rng.randint(0, W - 1, 2000) + 0.5, rng.randint(0, H - 1, 2000) + 0.5
    near, far = rng.uniform(3, 10, 2000), rng.uniform(20, 60, 2000)
    a, b = _from_pixels(k[0], k[1], near), _from_pixels(k[0], k[1], far)
    flip = rng.rand(2000) < 0.5
    first = np.where(flip[:, None], a, b)
    second = np.where(flip[:, None], b, a)
    outside = np.concatenate([_from_pixels(rng.uniform(-300, -1, 500), rng.uniform(0, H, 500), rng.uniform(5, 40, 500)),
                              _from_pixels(rng.uniform(0, W, 500), rng.uniform(H, H + 200, 500), rng.uniform(5, 40, 500))])
    behind = np.stack([rng.uniform(-20, 2, 1000), rng.uniform(-10, 10, 1000), rng.uniform(-2, 2, 1000)], 1)   # x <= 2
    xyz = np.concatenate([pts, first, outside, behind, second]).astype(np.float32)
    keep = ~near_boundary(xyz, H=H, W=W)
    xyz = xyz[keep]
    margin_pts = np.concatenate([xyz, rng.uniform(0, 1, (len(xyz), 1)).astype(np.float32)], 1)
    dense = np.concatenate([rng.uniform([-5, -40, -3], [80, 40, 3], (120000, 3)), rng.uniform(0, 1, (120000, 1))], 1).astype(np.float32)
    # KITTI-sized cloud: ~120k points, most of them out of view (as a 360-degree scan)
    base = dict(R0_rect=R0, Tr_velo_to_cam=TR, P2=P2, baseline=BASELINE, H=H, W=W)
    return [dict(base, id="margin", points=margin_pts, margin=True),
            dict(base, id="kitti_scan_120k", points=dense, margin=False)]


# ---- a small KITTI tree for the precompute CLI ---------------------------------------------------------------------------------------

TREE_SIZES = [(375, 1242), (370, 1224)]


def stereo_frame(seed, H, W, d):
    """An RGB pair whose right frame is the left shifted by d pixels (three textured channels)."""
    chans = [banded(seed + c, H, W, [(0, H, d)], sigma=1.5) for c in range(3)]
    return np.stack([c[0] for c in chans], 2), np.stack([c[1] for c in chans], 2)


def write_tree(tmp, sizes=TREE_SIZES, n_points=20000):
    """A KITTI training tree (image_2, image_3, calib, velodyne), the train / val split files and a Stereo3D-like config with the
    reference's test augmentation (CropTop 100, Resize to 288x1280, Normalize).  Returns the config's path."""
    import cv2
    raw = os.path.join(tmp, "kitti", "training")
    for d in ("calib", "image_2", "image_3", "velodyne"):
        os.makedirs(os.path.join(raw, d), exist_ok=True)
    names = []
    for i, (H, W) in enumerate(sizes):
        idx = "%06d" % (3 * i + 1)                                   # KITTI indices differ from the output numbering
        names.append(idx)
        left, right = stereo_frame(30 + 10 * i, H, W, 40 + 17 * (i % 8))
        cv2.imwrite(os.path.join(raw, "image_2", idx + ".png"), left)
        cv2.imwrite(os.path.join(raw, "image_3", idx + ".png"), right)
        fmt = lambda a: " ".join("%.12e" % v for v in np.asarray(a).reshape(-1))
        with open(os.path.join(raw, "calib", idx + ".txt"), "w") as f:
            f.write(f"P0: {fmt(P2)}\nP1: {fmt(P2)}\nP2: {fmt(P2)}\nP3: {fmt(P3)}\nR0_rect: {fmt(R0[:3, :3])}\n"
                    f"Tr_velo_to_cam: {fmt(TR[:3])}\nTr_imu_to_velo: {fmt(np.eye(3, 4))}\n")
        rng = np.random.RandomState(50 + i)
        pts = np.concatenate([rng.uniform([-5, -30, -3], [70, 30, 2], (n_points, 3)), rng.uniform(0, 1, (n_points, 1))], 1)
        pts.astype(np.float32).tofile(os.path.join(raw, "velodyne", idx + ".bin"))
    split = os.path.join(tmp, "split")
    os.makedirs(split, exist_ok=True)
    for name in ("train.txt", "val.txt"):
        with open(os.path.join(split, name), "w") as f:
            f.write("".join(n + "\n" for n in names))
    pre = os.path.join(tmp, "pre")
    os.makedirs(pre, exist_ok=True)
    cfg = os.path.join(tmp, "stereo_config.py")
    with open(cfg, "w") as f:
        f.write(f"""from easydict import EasyDict as edict
import numpy as np
cfg = edict()
cfg.trainer = edict(gpu=0)
cfg.path = edict(data_path={raw!r}, preprocessed_path={pre!r})
cfg.data = edict(train_split_file={os.path.join(split, 'train.txt')!r}, val_split_file={os.path.join(split, 'val.txt')!r})
cfg.data.augmentation = edict(rgb_mean=np.array([0.485, 0.456, 0.406]), rgb_std=np.array([0.229, 0.224, 0.225]), crop_top=100,
                              cropSize=(288, 1280))
cfg.data.test_augmentation = [
    edict(type_name='ConvertToFloat'),
    edict(type_name='CropTop', keywords=edict(crop_top_index=cfg.data.augmentation.crop_top)),
    edict(type_name='Resize', keywords=edict(size=cfg.data.augmentation.cropSize)),
    edict(type_name='Normalize', keywords=edict(mean=cfg.data.augmentation.rgb_mean, stds=cfg.data.augmentation.rgb_std)),
]
""")
    return cfg
