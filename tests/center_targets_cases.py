"""Constructed label sets for the KM3D / MonoFlex target encoder (visualdet3d_b200/center_targets.py), shared by
tests/golden/make_golden_center_targets.py and the tests.  Each case: detector mode, image size, P2 and a list of objects
(x, y, z, w, h, l, ry, bbox_l, bbox_t, bbox_r, bbox_b, class index).  Random objects are KITTI-like, with their 2-D box the hull of the
projected 3-D box; the generator nudges any object whose float32-projected coordinates come within 1e-3 heatmap px of an integer."""
import math

import numpy as np

OBJ_TYPES = ["Car", "Pedestrian", "Cyclist"]
P2_KITTI = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]])
# theta == 0 exactly (x + P2[0, 3] / P2[0, 0] == 0, ry == 0) and z + w / 2 == 32 (so z + 1e-6 rounds back to 32 in float32): corners 3 and
# 4 project to u = (10880 * 2 + 600 * 32) / 32 = 1280 exactly, i.e. x == hm_w at 384x1280, with no rounded trigonometry on the way.
P2_EXACT = np.array([[10880.0, 0.0, 600.0, 0.0], [0.0, 700.0, 180.0, 0.0], [0.0, 0.0, 1.0, 0.0]])
SIZES = [(384, 1280), (375, 1242)]


class Obj:
    __slots__ = ("x", "y", "z", "w", "h", "l", "ry", "bbox_l", "bbox_t", "bbox_r", "bbox_b", "type", "alpha")

    def __init__(self, v, cls):
        self.x, self.y, self.z, self.w, self.h, self.l, self.ry, self.bbox_l, self.bbox_t, self.bbox_r, self.bbox_b = [float(a) for a in v]
        self.type = OBJ_TYPES[cls]
        self.alpha = None


def corners(v, P2, nc):
    """float64 projection of the 3-D box (the reference's corner order; MonoFlex's rows 8-10 when nc == 11) -> image (u, v), camera z."""
    x, y, z, w, h, l, ry = v[:7]
    cm = np.array([[-1, -1, -1], [1, -1, -1], [1, 1, -1], [1, 1, 1], [1, -1, 1], [-1, -1, 1], [-1, 1, 1], [-1, 1, -1],
                   [0, 1, 0], [0, -1, 0], [0, 0, 0]], np.float64)
    if nc == 9:
        cm = np.concatenate([cm[:8], cm[10:]])
    theta = ry
    rel = 0.5 * cm * np.array([w, h, l])
    c, s = math.cos(theta), math.sin(theta)
    ax = rel[:, 2] * c + rel[:, 0] * s + x
    az = -rel[:, 2] * s + rel[:, 0] * c + z
    ay = rel[:, 1] + y - 0.5 * h
    cam = P2 @ np.stack([ax, ay, az, np.ones_like(ax)])
    return cam[0] / cam[2], cam[1] / cam[2], az


def random_obj(rng, P2, H, W, z_range=(5.0, 60.0), x_range=(-15.0, 15.0)):
    z = rng.uniform(*z_range)
    h, w, l = rng.uniform(1.4, 1.8), rng.uniform(1.5, 1.9), rng.uniform(3.5, 4.5)
    v = [rng.uniform(*x_range), rng.uniform(1.0, 2.0), z, w, h, l, rng.uniform(-math.pi, math.pi)]
    u, vv, _ = corners(v, P2, 9)
    j = rng.uniform(-3, 3, 4)
    return v + [u[:8].min() + j[0], vv[:8].min() + j[1], u[:8].max() + j[2], vv[:8].max() + j[3]]


def ry_for_alpha(alpha, x, z, P2):
    return alpha + math.atan2(x + P2[0, 3] / P2[0, 0], z)


def build_cases():
    """-> list of (name, mode, H, W, P2, [(row, cls)]); mode 0 KM3D, 1 MonoFlex."""
    rng = np.random.RandomState(7)
    cases = []

    def add(name, mode, H, W, P2, objs):
        cases.append((name, mode, H, W, P2, objs))

    for mode in (0, 1):
        H, W = SIZES[0]
        add("empty", mode, H, W, P2_KITTI, [])
        add("kitti6", mode, H, W, P2_KITTI, [(random_obj(rng, P2_KITTI, H, W), int(rng.randint(3))) for _ in range(6)])
        add("kitti12_375x1242", mode, *SIZES[1], P2_KITTI,
            [(random_obj(rng, P2_KITTI, *SIZES[1]), int(rng.randint(3))) for _ in range(12)])
        add("cap32", mode, H, W, P2_KITTI, [(random_obj(rng, P2_KITTI, H, W), int(rng.randint(3))) for _ in range(32)])
        add("over33", mode, H, W, P2_KITTI, [(random_obj(rng, P2_KITTI, H, W), 0) for _ in range(33)])
        edge = []
        base = random_obj(rng, P2_KITTI, H, W, z_range=(15, 20), x_range=(-1, 1))
        edge.append((base[:7] + [-80.0, 150.0, -8.0, 220.0], 0))                 # clipped bbox of zero width (left of the image)
        edge.append((base[:7] + [500.0, 390.0, 560.0, 420.0], 1))                # clipped bbox of zero height (below the image)
        edge.append((base[:7] + [400.0, 120.0, 480.0, 200.0], 0))                # KM3D centre exactly on an integer: (110, 40)
        edge.append((base[:7] + [600.0, 100.0, 602.0, 102.0], 2))                # 2x2 px box: radius 0
        edge.append((base[:7] + [1281.0, 100.0, 1400.0, 200.0], 0))              # starts beyond the right edge: zero width
        for alpha in (math.pi / 6 - 0.02, math.pi / 6 + 0.02, -math.pi / 6 - 0.02, -math.pi / 6 + 0.02,
                      5 * math.pi / 6 - 0.02, 5 * math.pi / 6 + 0.02, -5 * math.pi / 6 + 0.02, -5 * math.pi / 6 - 0.02):
            o = random_obj(rng, P2_KITTI, H, W, z_range=(10, 40), x_range=(-8, 8))
            o[6] = ry_for_alpha(alpha, o[0], o[2], P2_KITTI)                   # sin(alpha) on both sides of +-0.5
            edge.append((o, int(rng.randint(3))))
        near = random_obj(rng, P2_KITTI, H, W, z_range=(12, 14), x_range=(0.5, 1.0))
        edge.append((near, 1))
        twin = list(near)
        twin[0] += 0.37
        twin[7] += 10.3
        twin[9] += 10.3
        edge.append((twin, 1))                                                  # an overlapping object of the same class
        add("edges", mode, H, W, P2_KITTI, edge)
        big = []
        # large, near objects at the four borders: their keypoints leave the map or sit on its edges, their splats are clipped
        for x, y, z, ry in ((-4.6, 1.7, 5.5, 0.3), (4.4, 1.7, 5.2, -0.4), (-1.3, 1.7, 4.0, 1.2), (0.9, 1.7, 3.1, 2.9), (0.5, 0.7, 4.0, 0.3)):
            o = [x, y, z, 1.8, 1.6, 4.2, ry]
            u, v, _ = corners(o, P2_KITTI, 9)
            big.append((o + [u.min() - 10, v.min() - 10, u.max() + 10, v.max() + 10], 0))
        # behind the camera: corners with z < 0 (MonoFlex's visibility), projected far outside the map
        big.append(([2.0, 1.6, 1.2, 1.7, 1.5, 4.0, 0.25, 700.0, 150.0, 1279.0, 383.0], 0))
        big.append(([-3.0, 1.6, 0.9, 1.7, 1.5, 4.0, 1.9, 0.0, 150.0, 500.0, 383.0], 2))
        big.append(([0.1, 0.85, 1.5, 1.7, 1.5, 4.0, 1.4, 0.0, 0.0, 1279.0, 383.0], 1))          # ... with its centre in the map
        # MonoFlex: a projected centre in (-1, 0) and one beyond hm_w; keypoints in (-1, 0) for KM3D
        for uc in (-2.5, 1285.0, 3.0):
            z = 20.0
            x = ((uc * (z + P2_KITTI[2, 3]) - P2_KITTI[0, 2] * z - P2_KITTI[0, 3]) / P2_KITTI[0, 0])
            big.append(([x, 1.6, z, 1.7, 1.5, 4.0, ry_for_alpha(0.3, x, z, P2_KITTI), 0.0, 150.0, max(uc, 0.0) + 60.0, 230.0], 1))
        add("borders", mode, H, W, P2_KITTI, big)
        # a keypoint exactly at x == hm_w (MonoFlex: visible, yet no heatmap, offset or index)
        add("exact_hm_w", mode, H, W, P2_EXACT, [([0.0, 1.0, 31.0, 2.0, 1.5, 4.0, 0.0, 500.0, 150.0, 700.0, 250.0], 0)])
    return cases
