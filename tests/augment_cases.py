"""Constructed frames and descriptors for the augmentation kernel (visualdet3d_b200/csrc/train_augment.cu), for training and as the
test-time resize, built directly rather than through TrainAugmentation's random draws.  Used by tests/golden/make_golden_augment_cases.py
(the cv2 / numpy expectation), tests/test_augment_cases_cpu.py and tests/test_augment_cases_gpu.py.

Every case is a dict: id, group ("resize" geometry only, "warp", or "colour" for a photometric program), the uint8 HWC frame, geom, crop_top,
the forward 2x3 affine (float32), mirror, the op codes / float32 args / float64 noise of the photometric program, and the output Ho x Wo.
`closed_form(case)` gives the float64 network input where one exists: impulse and ramp frames through the resize (bilinear interpolation of
a linear function is linear, clamped coordinates included) and warps whose inverse map is integral (identity, integer shifts, the 90 degree
rotation, a map that sends every output outside the frame).  Nothing here imports the package: the fixture generator uses it too."""
import math

import numpy as np

MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)
GEOM_RESIZE, GEOM_WARP_U8, GEOM_WARP_F32 = 0, 1, 2
OP_BRIGHTNESS, OP_CONTRAST, OP_RGB2HSV, OP_SATURATION, OP_HUE, OP_HSV2RGB, OP_EIGEN_NOISE = range(1, 8)
IDENTITY = np.array([[1, 0, 0], [0, 1, 0]], np.float32)

# the kernel's tile and the resize step describe() accepts (train_augment.cu: AUG_TX, AUG_RY, AUG_MAX_SCALE)
TILE_X, TILE_Y, MAX_SCALE = 128, 4, 2
GEOMETRY_TOL, COLOUR_TOL = 2e-6, 5e-5


# ---- the resize geometry, restated ------------------------------------------------------------------------------------------------------
def resize_geom(Hc, W, Ho):
    """Resize(preserve_aspect_ratio) of an Hc x W frame to Ho rows: (Hr, Wr, scale_y, scale_x), cv2's source step per axis."""
    sf = Ho / Hc
    Hr, Wr = int(np.round(Hc * sf)), int(np.round(W * sf))
    return Hr, Wr, 1.0 / (Hr / Hc), 1.0 / (Wr / W)


def lin_coord(d, scale, n):
    """cv2.resize INTER_LINEAR: source index and weight of destination index d, clamped at the borders."""
    fd = (d + 0.5) * scale - 0.5
    s = math.floor(fd)
    f = fd - s
    if s < 0:
        s, f = 0, 0.0
    if s >= n - 1:
        s, f = n - 1, 0.0
    return s, f


def geometry(case):
    H, W = case["frame"].shape[:2]
    Hc = H - case["crop_top"]
    Hr, Wr, sy, sx = resize_geom(Hc, W, case["Ho"])
    return Hc, W, Wr, sy, sx


def tile_grid(case):
    return -(-case["Wo"] // TILE_X), -(-case["Ho"] // TILE_Y)


def stage_window(case, bx, by):
    """The source window (r0, r1, c0, c1), inclusive and in cropped-frame rows, that kernel tile (bx, by) stages in shared memory; None
    for a tile wholly in the zero pad.  A restatement of the kernel's window arithmetic (train_augment.cu, train_augment_kernel)."""
    Hc, W, Wr, sy, sx = geometry(case)
    Ho, Wo = case["Ho"], case["Wo"]
    x0, y0 = bx * TILE_X, by * TILE_Y
    x1, y1 = min(x0 + TILE_X, Wo) - 1, min(y0 + TILE_Y, Ho) - 1
    ul, uh = (Wo - 1 - x1, Wo - 1 - x0) if case["mirror"] else (x0, x1)
    uh = min(uh, Wr - 1)
    if ul > uh:
        return None
    r0, r1 = lin_coord(y0, sy, Hc)[0], lin_coord(y1, sy, Hc)[0]
    c0, c1 = lin_coord(ul, sx, W)[0], lin_coord(uh, sx, W)[0]
    return r0, min(r1 + 1, Hc - 1), c0, min(c1 + 1, W - 1)


# ---- case construction ------------------------------------------------------------------------------------------------------------------
def _case(cid, group, frame, Ho, Wo, geom=GEOM_RESIZE, crop_top=0, affine=IDENTITY, mirror=0, program=(), noise=(0.0, 0.0, 0.0), closed=None):
    return {"id": cid, "group": group, "frame": np.ascontiguousarray(frame, dtype=np.uint8), "geom": geom, "crop_top": crop_top,
            "affine": np.ascontiguousarray(affine, dtype=np.float32), "mirror": mirror,
            "ops": np.array([o for o, _ in program], np.int32), "args": np.array([a for _, a in program], np.float32),
            "noise": np.array(noise, np.float64), "Ho": Ho, "Wo": Wo, "closed": closed}


def _impulse_frame(H, W, crop_top, impulses):
    """Zeros with one RGB value per impulse at (cropped row, column)."""
    f = np.zeros((H, W, 3), np.uint8)
    for r, c, rgb in impulses:
        f[r + crop_top, c] = rgb
    return f


def _ramp_frame(H, W, a, b, axis, seed=None, crop_top=0):
    """value = a + b * column (axis 1) or a + b * row (axis 0) in every channel; rows above crop_top hold noise when seeded."""
    idx = np.arange(W if axis == 1 else H, dtype=np.float64)
    v = a + b * idx
    assert v.min() >= 0 and v.max() <= 255 and np.array_equal(v, np.round(v))
    f = np.broadcast_to((v[None, :, None] if axis == 1 else v[:, None, None]), (H, W, 3)).astype(np.uint8).copy()
    if seed is not None and crop_top:
        f[:crop_top] = np.random.RandomState(seed).randint(0, 256, (crop_top, W, 3))
    return f


IMPULSE_RGB = ((255, 100, 1), (37, 250, 128))


def _impulse_cases():
    """Impulses on the first and last staged row and column of chosen tiles, mirror off and on: an interior tile and the tile where Wr ends
    (partly pad), at an exact 2x source step, a step just under 2, and a strong upscale."""
    out = []
    Ho, Wo = 288, 400
    for step, H, W in (("2x", 576, 600), ("under2x", 575, 600), ("up", 37, 40)):
        for mirror in (0, 1):
            probe = _case("", "resize", np.zeros((H, W, 3), np.uint8), Ho, Wo, mirror=mirror)
            Wr = geometry(probe)[2]
            interior = 1                                                   # u 128..255 (mirror off), 271..144 (mirror on): inside Wr
            partial = (Wo - Wr if mirror else Wr - 1) // TILE_X            # the tile that holds the last resized column
            rows = (35, 35) if step != "up" else (0, tile_grid(probe)[1] - 1)
            for edge in ("first", "last"):
                by = rows[0] if edge == "first" else rows[1]
                imps = []
                for bx, rgb in zip((interior, partial), IMPULSE_RGB):
                    r0, r1, c0, c1 = stage_window(probe, bx, by)
                    imps.append((r0, c0, rgb) if edge == "first" else (r1, c1, rgb))
                out.append(_case(f"impulse_{step}_{edge}_m{mirror}", "resize", _impulse_frame(H, W, 0, imps), Ho, Wo, mirror=mirror,
                                 closed=("impulse", imps)))
    return out


def _ramp_cases():
    out = []
    # (id, H, W, crop_top, Ho, Wo, a, b, axis, mirrors)
    for cid, H, W, crop, Ho, Wo, a, b, axis, mirrors in (
            ("ramp_col_up", 30, 17, 0, 288, 170, 5, 15, 1, (0, 1)),         # 9.6x upscale, Wr = 163: a 7-column pad
            ("ramp_row_up_wr_eq_wo", 200, 50, 8, 288, 75, 0, 1, 0, (0,)),  # Wr == Wo
            ("ramp_row_down_wo_plus1", 250, 40, 0, 128, 21, 0, 1, 0, (0, 1)),   # a 1.95 step, Wr = 20: one pad column
            ("ramp_col_wo_minus1", 100, 200, 0, 60, 119, 20, 1, 1, (0, 1)),     # Wr = 120 cropped to 119
            ("ramp_col_pad_tiles", 100, 250, 0, 150, 520, 0, 1, 1, (0, 1)),     # Wr = 375 ends inside a tile, a tile wholly in the pad,
                                                                                 # Ho % 4 = 2, Wo % 128 = 8
            ("one_row_crop", 5, 3, 4, 16, 50, 40, 80, 1, (0, 1)),               # crop_top = H - 1: a one-row source
            ("one_col", 40, 1, 0, 80, 5, 0, 5, 0, (0, 1)),                      # a one-column source, Wr = 2
            ("three_col", 60, 3, 0, 100, 4, 10, 100, 1, (0, 1))):               # Wr = 5 cropped to 4
        for m in mirrors:
            f = _ramp_frame(H, W, a, b, axis, seed=H * W, crop_top=crop)
            out.append(_case(f"{cid}_m{m}", "resize", f, Ho, Wo, crop_top=crop, mirror=m, closed=("ramp", a, b, axis)))
    return out


def _warp_cases():
    frame = np.random.RandomState(11).randint(0, 256, (37, 53, 3)).astype(np.uint8)
    t = 33 / 2048          # inverse offset -16.5 / 1024: round-half-even and round-half-away put the fixed-point coordinate in different 1/32 cells
    out = []
    # (id, forward matrix, Ho, Wo, mirror, integral inverse map)
    for cid, M, Ho, Wo, m, exact in (
            ("identity", [[1, 0, 0], [0, 1, 0]], 40, 60, 0, True),           # the output overhangs the frame: zeros right and below
            ("shift_int", [[1, 0, 3], [0, 1, -2]], 40, 60, 0, True),
            ("shift_int_neg", [[1, 0, -5], [0, 1, 4]], 40, 60, 1, True),
            ("shift_half", [[1, 0, 0.5], [0, 1, -0.5]], 37, 53, 0, False),   # taps at -1 on the left, one past the bottom
            ("shift_half_neg", [[1, 0, -0.5], [0, 1, 0.5]], 37, 53, 0, False),   # taps one past the right, at -1 on the top
            ("shift_straddle", [[1, 0, -3.25], [0, 1, 2.75]], 40, 60, 0, False),
            ("rot90", [[0, 1, 0], [-1, 0, 52]], 53, 37, 0, True),
            ("zoom2", [[2, 0, -10.3], [0, 2, -7.1]], 40, 60, 0, False),
            ("zoom_half", [[0.5, 0, 0], [0, 0.5, 0]], 40, 60, 1, False),
            ("all_outside", [[1, 0, 100], [0, 1, 0]], 40, 60, 0, True),
            ("tie_1_2048", [[1, 0, 1 / 2048], [0, 1, 3 / 2048]], 40, 60, 0, False),
            ("tie_33_2048", [[1, 0, t], [0, 1, t]], 40, 60, 0, False),
            ("tie_33_2048_m", [[1, 0, -t], [0, 1, t]], 40, 60, 1, False)):
        for geom in (GEOM_WARP_U8, GEOM_WARP_F32):
            out.append(_case(f"warp_{'u8' if geom == GEOM_WARP_U8 else 'f32'}_{cid}", "warp", frame, Ho, Wo, geom=geom,
                             affine=np.array(M, np.float32), mirror=m, closed=("map",) if exact else None))
    # KM3D's order: the warp on the float32 frame, then a program with eigenvalue noise
    out.append(_case("warp_f32_program", "colour", frame, 40, 60, geom=GEOM_WARP_F32, affine=np.array([[1.3, 0.1, -4.6], [-0.05, 1.2, -2.2]], np.float32),
                     mirror=1, program=[(OP_BRIGHTNESS, 21.5), (OP_RGB2HSV, 0), (OP_SATURATION, 1.25), (OP_HSV2RGB, 0), (OP_CONTRAST, 0.8),
                                        (OP_EIGEN_NOISE, 0)], noise=(4.25, -2.5, 1.125)))
    return out


# The photometric palette: each column one colour (row 1 repeats row 0 in reverse order).
PALETTE = np.array(
    [(0, 0, 0), (1, 1, 1), (128, 128, 128), (254, 254, 254), (255, 255, 255),                       # greys: s == 0
     (255, 0, 0), (255, 255, 0), (0, 255, 0), (0, 255, 255), (0, 0, 255), (255, 0, 255),            # hue 0, 60, ..., 300
     (200, 200, 10), (10, 200, 200), (200, 10, 200), (5, 5, 4), (4, 5, 5), (5, 4, 5),               # ties for the maximum channel
     (5, 4, 4), (4, 5, 4), (4, 4, 5), (255, 254, 254), (254, 255, 255), (1, 0, 0),                  # near-greys, a difference of 1
     (10, 0, 3), (10, 3, 0),                                                                        # hue exactly 342 and 18: +-18 lands on 360 / 0
     (10, 0, 2), (10, 2, 0), (10, 4, 0), (0, 10, 1),                                                # hue 348, 12, 24, 126: +-18 crosses or stays
     (3, 0, 0), (20, 30, 10), (250, 3, 1), (1, 3, 250), (255, 1, 0), (255, 0, 1),                    # brightness -32 drives below 0
     (240, 250, 230), (230, 240, 255), (128, 64, 32)], np.uint8)                                    # +32 drives above 255

PROGRAMS = (
    ("hsv_round_trip", [(OP_RGB2HSV, 0), (OP_HSV2RGB, 0)]),
    ("hsv_only", [(OP_RGB2HSV, 0)]),                                       # the HSV values themselves reach Normalize
    ("hue_p18_hsv", [(OP_RGB2HSV, 0), (OP_HUE, 18.0)]),
    ("hue_m18_hsv", [(OP_RGB2HSV, 0), (OP_HUE, -18.0)]),
    ("hue_p18", [(OP_RGB2HSV, 0), (OP_HUE, 18.0), (OP_HSV2RGB, 0)]),
    ("hue_m18", [(OP_RGB2HSV, 0), (OP_HUE, -18.0), (OP_HSV2RGB, 0)]),
    ("hue_m60_hsv", [(OP_RGB2HSV, 0), (OP_HUE, -60.0)]),                   # a tie's hue of 60 -/+ 1 ulp wraps to ~360 or stays at ~0
    ("saturation_0", [(OP_RGB2HSV, 0), (OP_SATURATION, 0.0), (OP_HSV2RGB, 0)]),
    ("saturation_1p5", [(OP_RGB2HSV, 0), (OP_SATURATION, 1.5), (OP_HSV2RGB, 0)]),
    ("contrast_first", [(OP_BRIGHTNESS, 32.0), (OP_CONTRAST, 1.4), (OP_RGB2HSV, 0), (OP_SATURATION, 0.7), (OP_HUE, -11.5), (OP_HSV2RGB, 0)]),
    ("contrast_last", [(OP_BRIGHTNESS, -32.0), (OP_RGB2HSV, 0), (OP_SATURATION, 1.3), (OP_HUE, 13.25), (OP_HSV2RGB, 0), (OP_CONTRAST, 0.6)]),
    ("eigen_noise", [(OP_BRIGHTNESS, -20.0), (OP_RGB2HSV, 0), (OP_HSV2RGB, 0), (OP_EIGEN_NOISE, 0)]),
)


def palette_frame():
    return np.stack([PALETTE, PALETTE[::-1]])


def _colour_cases():
    out = []
    for name, prog in PROGRAMS:
        noise = (3.2, -1.7, 0.4) if name == "eigen_noise" else (0.0, 0.0, 0.0)
        f = palette_frame()
        out.append(_case(f"colour_{name}", "colour", f, f.shape[0], f.shape[1], program=prog, noise=noise))   # identity geometry
    # the program on source pixels ahead of a mirrored, 1.875x downscale through the kernel's stage
    f = np.random.RandomState(5).randint(0, 256, (120, 90, 3)).astype(np.uint8)
    out.append(_case("resize_program_m1", "colour", f, 64, 50, mirror=1, program=PROGRAMS[9][1]))
    return out


CASES = _impulse_cases() + _ramp_cases() + _warp_cases() + _colour_cases()
BY_ID = {c["id"]: c for c in CASES}
assert len(BY_ID) == len(CASES)

# 577 x 101 with crop_top 1 -> 288 rows: scale_y is exactly 2 but Wr = round(50.5) = 50 makes scale_x 2.02, beyond the kernel's stage
REFUSED = {"H": 577, "W": 101, "crop_top": 1, "Ho": 288, "Wo": 60}


def tol(case):
    return COLOUR_TOL if case["group"] == "colour" else GEOMETRY_TOL


# ---- closed forms (float64) -------------------------------------------------------------------------------------------------------------
def normalize64(img):
    """[Ho, Wo, 3] float64 before Normalize -> [3, Ho, Wo] float64 network input."""
    out = (img / 255.0 - MEAN.astype(np.float64)) / STD.astype(np.float64)
    return np.ascontiguousarray(out.transpose(2, 0, 1))


def _clamped_coord(n_out, scale, n_src):
    d = np.arange(n_out, dtype=np.float64)
    return np.clip((d + 0.5) * scale - 0.5, 0.0, n_src - 1)


def inverse_map(affine):
    """cv2.warpAffine's destination -> source map of the float32 forward matrix, in float64."""
    M = affine.astype(np.float64)
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    A = np.array([[M[1, 1], -M[0, 1]], [-M[1, 0], M[0, 0]]]) / D
    return np.concatenate([A, -A @ M[:, 2:3]], axis=1)


def closed_form(case):
    """The float64 network input [3, Ho, Wo] of a case with a closed form, else None."""
    kind = case["closed"]
    if kind is None:
        return None
    Ho, Wo = case["Ho"], case["Wo"]
    img = np.zeros((Ho, Wo, 3))
    if kind[0] in ("impulse", "ramp"):
        Hc, W, Wr, sy, sx = geometry(case)
        n = min(Wr, Wo)
        cy, cx = _clamped_coord(Ho, sy, Hc), _clamped_coord(n, sx, W)
        if kind[0] == "impulse":
            for r, c, rgb in kind[1]:
                w = np.maximum(0.0, 1.0 - np.abs(cy - r))[:, None] * np.maximum(0.0, 1.0 - np.abs(cx - c))[None, :]
                img[:, :n] += w[:, :, None] * np.array(rgb, np.float64)
        else:
            _, a, b, axis = kind
            v = a + b * (cx[None, :] if axis == 1 else (cy[:, None] + case["crop_top"]))
            img[:, :n] = np.broadcast_to(v, (Ho, n))[:, :, None]
    else:
        A = inverse_map(case["affine"])
        y, x = np.mgrid[0:Ho, 0:Wo].astype(np.float64)
        sx, sy = A[0, 0] * x + A[0, 1] * y + A[0, 2], A[1, 0] * x + A[1, 1] * y + A[1, 2]
        assert np.array_equal(sx, np.round(sx)) and np.array_equal(sy, np.round(sy)), case["id"]
        H, W = case["frame"].shape[:2]
        sx, sy = sx.astype(np.int64), sy.astype(np.int64)
        inside = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H)
        img[inside] = case["frame"][sy[inside], sx[inside]]
    if case["mirror"]:
        img = img[:, ::-1]
    return normalize64(img)
