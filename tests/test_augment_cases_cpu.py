"""The augmentation's host form (`vd3d_train_augment_host`), for training and as the test-time resize (`preprocess_host`), on the
constructed cases of tests/augment_cases.py, without a GPU:
  * against the cv2 / numpy fixture (tests/golden/make_golden_augment_cases.py): 2e-6 on geometry, 5e-5 on colour programs;
  * against float64 closed forms on the impulse, ramp, integral-warp and all-outside cases;
  * the case set reaches what it is meant to: impulses on the first and last staged row and column at the exact 2x step (mirror off and on),
    a tile wholly in the pad, partial border taps, grey pixels, each tie for the maximum channel, hues landing on 0 and 360, wraps both ways;
  * sensitivity: a float32 numpy restatement of the per-pixel routine, including the kernel's shared-memory window, matches the fixture; each
    perturbation of it (a window one row / column short, no border clamp, a float32 coordinate, `>=` in the hue wrap, `v == g` tested first,
    round-half-away in the warp, `>> 10` without `+ 512`) moves at least one case beyond the tolerance, so a kernel or host form making that
    mistake fails here or in tests/test_augment_cases_gpu.py;
  * the refusal boundary of the kernel's 2x stage."""
import numpy as np
import pytest

import augment_cases as ac
from conftest import GOLDEN
from visualdet3d_b200 import _lib
from visualdet3d_b200 import preprocess as pp
from visualdet3d_b200 import train_augment as ta

F32 = np.float32
EPS = F32(np.finfo(np.float32).eps)


def _fixture():
    return np.load(f"{GOLDEN}/augment_cases.npz")


def deferred(c):
    return ta.DeferredFrame(c["frame"], c["geom"], c["crop_top"], c["affine"], c["mirror"], c["ops"], c["args"], c["noise"], c["Ho"], c["Wo"],
                            ac.MEAN, ac.STD)


def plain_resize(c):
    """A resize case with no program: the test-time pipeline computes the same image before the mirror."""
    return c["geom"] == ac.GEOM_RESIZE and len(c["ops"]) == 0


# ---- the float32 restatement of aug_pixel ------------------------------------------------------------------------------------------------
def rgb_to_hsv(c, g_first=False, trace=None):
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    v = np.maximum(np.maximum(r, g), b)
    vmin = np.minimum(np.minimum(r, g), b)
    diff = v - vmin
    s = diff / (np.abs(v) + EPS)
    diff = F32(60) / (diff + EPS)
    hr, hg, hb = (g - b) * diff, (b - r) * diff + F32(120), (r - g) * diff + F32(240)
    if g_first:
        h = np.where(v == g, hg, np.where(v == r, hr, hb))
    else:
        h = np.where(v == r, hr, np.where(v == g, hg, hb))
    h = np.where(h < 0, h + F32(360), h)
    if trace is not None:
        for name, m in (("tie_rg", (r == g) & (g > b)), ("tie_gb", (g == b) & (b > r)), ("tie_rb", (r == b) & (b > g))):
            if m.any():
                trace.add(name)
    return np.stack([h, s, v], -1)


# cv2's sector table: the (b, g, r) entries of {v, v(1-s), v(1-sh), v(1-s(1-h))} per sector
SECTOR_BGR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def hsv_to_rgb(c, drop_s0=False, trace=None):
    h, s, v = c[..., 0], c[..., 1], c[..., 2]
    hh = np.fmod(h * (F32(6) / F32(360)), F32(6))
    hh = np.where(hh < 0, hh + F32(6), hh)
    sector = np.floor(hh).astype(np.int64)
    hh = hh - sector.astype(F32)
    bad = (sector < 0) | (sector >= 6)
    sector, hh = np.where(bad, 0, sector), np.where(bad, F32(0), hh)
    tab = np.stack([v, v * (F32(1) - s), v * (F32(1) - s * hh), v * (F32(1) - s * (F32(1) - hh))], -1)
    bgr = np.take_along_axis(tab, SECTOR_BGR[sector], -1)
    rgb = bgr[..., ::-1]
    if trace is not None and (s == 0).any():
        trace.add("s_zero")
    if not drop_s0:
        rgb = np.where((s == 0)[..., None], v[..., None], rgb)
    return rgb


def apply_program(c, case, ge_wrap=False, g_first=False, drop_s0=False, trace=None):
    c = c.astype(F32)
    for op, a in zip(case["ops"], case["args"]):
        if op == ac.OP_BRIGHTNESS:
            c = c + a
        elif op == ac.OP_CONTRAST:
            c = c * a
        elif op == ac.OP_RGB2HSV:
            c = rgb_to_hsv(c, g_first, trace)
        elif op == ac.OP_SATURATION:
            c = c.copy()
            c[..., 1] = c[..., 1] * a
        elif op == ac.OP_HUE:
            c = c.copy()
            h = c[..., 0] + a
            if trace is not None:
                for name, m in (("hue_at_360", h == 360), ("hue_at_0", h == 0), ("wrap_down", h > 360), ("wrap_up", h < 0)):
                    if m.any():
                        trace.add(name)
            h = np.where((h >= 360) if ge_wrap else (h > 360), h - F32(360), h)
            c[..., 0] = np.where(h < 0, h + F32(360), h)
        elif op == ac.OP_HSV2RGB:
            c = hsv_to_rgb(c, drop_s0, trace)
        elif op == ac.OP_EIGEN_NOISE:
            c = (c.astype(np.float64) + case["noise"]).astype(F32)
    return c


def _lin(d, scale, n, clamp=True, f32_coord=False):
    fd = (d + 0.5) * scale - 0.5
    if f32_coord:
        fd = fd.astype(F32).astype(np.float64)
    s = np.floor(fd).astype(np.int64)
    f = (fd - s).astype(F32)
    if clamp:
        f = np.where((s < 0) | (s >= n - 1), F32(0), f)
        s = np.clip(s, 0, n - 1)
    return s, f


def restate_resize(case, shrink=None, clamp=True, f32_coord=False, trace=None, **prog):
    """[Ho, Wo, 3] before Normalize, read through the kernel's per-tile stage.  `shrink` ("top", "bottom", "left" or "right"): every tile's
    window one row / column short on that side.  A tap outside the window or the frame reads 0."""
    Hc, W, Wr, sy, sx = ac.geometry(case)
    Ho, Wo = case["Ho"], case["Wo"]
    src = apply_program(case["frame"][case["crop_top"]:], case, trace=trace, **prog)
    y, x = np.arange(Ho)[:, None], np.arange(Wo)[None, :]
    u = Wo - 1 - x if case["mirror"] else x
    r, fy = _lin(y, sy, Hc, clamp, f32_coord)
    c, fx = _lin(np.minimum(u, Wr - 1), sx, W, clamp, f32_coord)
    r1, c1 = np.where(r + 1 < Hc, r + 1, r), np.where(c + 1 < W, c + 1, c)
    lo_r, hi_r, lo_c, hi_c = (np.zeros((Ho, Wo), np.int64) for _ in range(4))
    nbx, nby = ac.tile_grid(case)
    for by in range(nby):
        for bx in range(nbx):
            w = ac.stage_window(case, bx, by)
            if w is None:
                continue
            r0, rr1, c0, cc1 = w
            if shrink:
                r0, rr1, c0, cc1 = r0 + (shrink == "top"), rr1 - (shrink == "bottom"), c0 + (shrink == "left"), cc1 - (shrink == "right")
            sl = np.s_[by * ac.TILE_Y:(by + 1) * ac.TILE_Y, bx * ac.TILE_X:(bx + 1) * ac.TILE_X]
            lo_r[sl], hi_r[sl], lo_c[sl], hi_c[sl] = r0, rr1, c0, cc1

    def tap(rr, cc):
        ok = (rr >= lo_r) & (rr <= hi_r) & (cc >= lo_c) & (cc <= hi_c) & (rr >= 0) & (rr < Hc) & (cc >= 0) & (cc < W)
        return np.where(ok[..., None], src[np.clip(rr, 0, Hc - 1), np.clip(cc, 0, W - 1)], F32(0))

    a0, a1, b0, b1 = (F32(1) - fx)[..., None], fx[..., None], (F32(1) - fy)[..., None], fy[..., None]
    h0 = tap(r, c) * a0 + tap(r, c1) * a1
    h1 = tap(r1, c) * a0 + tap(r1, c1) * a1
    v = h0 * b0 + h1 * b1
    return np.where((u < Wr)[..., None], v, F32(0))


def _round_half_away(v):
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)


def restate_warp(case, half_away=False, no_plus512=False, trace=None, **prog):
    m = ac.inverse_map(case["affine"]).reshape(-1)
    rnd = _round_half_away if half_away else (lambda t: np.rint(t).astype(np.int64))
    H, W = case["frame"].shape[:2]
    Ho, Wo = case["Ho"], case["Wo"]
    y, x = np.arange(Ho, dtype=np.float64)[:, None], np.arange(Wo)[None, :]
    u = (Wo - 1 - x if case["mirror"] else x).astype(np.float64)
    X = (rnd((m[1] * y + m[2]) * 1024) + 16 + rnd(m[0] * u * 1024)) >> 5
    Y = (rnd((m[4] * y + m[5]) * 1024) + 16 + rnd(m[3] * u * 1024)) >> 5
    sx, sy, fx, fy = X >> 5, Y >> 5, X & 31, Y & 31
    taps, inside = [], []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        rr, cc = sy + dy, sx + dx
        ok = (rr >= 0) & (rr < H) & (cc >= 0) & (cc < W)
        taps.append(np.where(ok[..., None], case["frame"][np.clip(rr, 0, H - 1), np.clip(cc, 0, W - 1)], 0).astype(np.int64))
        inside.append(ok)
    if trace is not None and (np.any(inside, 0) & ~np.all(inside, 0)).any():
        trace.add("partial_border_taps")
    if case["geom"] == ac.GEOM_WARP_U8:
        w = [(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx]
        s = sum(t * wi[..., None] for t, wi in zip(taps, w))
        v = ((s if no_plus512 else s + 512) >> 10).astype(F32)
    else:
        wx, wy = fx.astype(F32) * F32(1 / 32), fy.astype(F32) * F32(1 / 32)
        w = [(F32(1) - wy) * (F32(1) - wx), (F32(1) - wy) * wx, wy * (F32(1) - wx), wy * wx]
        t = [tt.astype(F32) for tt in taps]
        v = t[0] * w[0][..., None] + t[1] * w[1][..., None] + t[2] * w[2][..., None] + t[3] * w[3][..., None]
    return apply_program(v, case, trace=trace, **prog)


def restate(case, shrink=None, clamp=True, f32_coord=False, half_away=False, no_plus512=False, trace=None, **prog):
    """The float32 restatement of the network input [3, Ho, Wo]; the keywords select a perturbation."""
    if case["geom"] == ac.GEOM_RESIZE:
        img = restate_resize(case, shrink, clamp, f32_coord, trace, **prog)
    else:
        img = restate_warp(case, half_away, no_plus512, trace, **prog)
    img = (img / F32(255.0) - ac.MEAN) / ac.STD
    return np.ascontiguousarray(img.transpose(2, 0, 1))


# ---- the host forms against the fixture and the closed forms ------------------------------------------------------------------------------
def test_host_form_matches_fixture():
    fx = _fixture()
    worst = {}
    for c in ac.CASES:
        d = float(np.abs(ta.augment_host(deferred(c)) - fx[c["id"]]).max())
        worst[c["group"]] = max(worst.get(c["group"], 0.0), d)
        assert d <= ac.tol(c), (c["id"], d)
    print("host form vs cv2 fixture, max |diff| per group: " + ", ".join(f"{g} {d:.2e}" for g, d in worst.items()))


def test_preprocess_host_matches_fixture_on_resize_cases():
    fx = _fixture()
    n, worst = 0, 0.0
    for c in ac.CASES:
        if not plain_resize(c):
            continue
        got = pp.preprocess_host(c["frame"], c["crop_top"], (c["Ho"], c["Wo"]), ac.MEAN, ac.STD)
        want = fx[c["id"]][:, :, ::-1] if c["mirror"] else fx[c["id"]]
        d = float(np.abs(got - want).max())
        worst, n = max(worst, d), n + 1
        assert d <= ac.GEOMETRY_TOL, (c["id"], d)
    assert n >= 20
    print(f"preprocess host form vs cv2 fixture on {n} resize cases: max |diff| {worst:.2e}")


@pytest.mark.parametrize("case", [c for c in ac.CASES if c["closed"]], ids=[c["id"] for c in ac.CASES if c["closed"]])
def test_closed_forms(case):
    want = ac.closed_form(case)
    assert float(np.abs(_fixture()[case["id"]] - want).max()) <= ac.GEOMETRY_TOL       # the fixture itself
    assert float(np.abs(ta.augment_host(deferred(case)) - want).max()) <= ac.GEOMETRY_TOL
    if plain_resize(case):
        got = pp.preprocess_host(case["frame"], case["crop_top"], (case["Ho"], case["Wo"]), ac.MEAN, ac.STD)
        assert float(np.abs(got - (want[:, :, ::-1] if case["mirror"] else want)).max()) <= ac.GEOMETRY_TOL


# ---- coverage -------------------------------------------------------------------------------------------------------------------------
def test_impulses_sit_on_every_edge_of_the_stage_at_the_2x_step():
    seen = set()
    for c in ac.CASES:
        if not c["closed"] or c["closed"][0] != "impulse":
            continue
        Hc, W, Wr, sy, sx = ac.geometry(c)
        if not (sy == 2.0 and sx == 2.0):
            continue
        nbx, nby = ac.tile_grid(c)
        for r, col, _ in c["closed"][1]:
            for by in range(nby):
                for bx in range(nbx):
                    w = ac.stage_window(c, bx, by)
                    if w is None or not (w[0] <= r <= w[1] and w[2] <= col <= w[3]):
                        continue
                    for edge, hit in (("first_row", r == w[0]), ("last_row", r == w[1]), ("first_col", col == w[2]), ("last_col", col == w[3])):
                        if hit:
                            seen.add((edge, c["mirror"]))
    assert seen == {(e, m) for e in ("first_row", "last_row", "first_col", "last_col") for m in (0, 1)}, seen


def test_cases_reach_every_branch():
    trace = set()
    pad_tiles = set()
    for c in ac.CASES:
        restate(c, trace=trace)
        if c["geom"] == ac.GEOM_RESIZE:
            nbx, nby = ac.tile_grid(c)
            if any(ac.stage_window(c, bx, 0) is None for bx in range(nbx)):
                pad_tiles.add(c["mirror"])
    want = {"s_zero", "tie_rg", "tie_gb", "tie_rb", "hue_at_0", "hue_at_360", "wrap_down", "wrap_up", "partial_border_taps"}
    assert want <= trace, want - trace
    assert pad_tiles == {0, 1}
    # the window never exceeds the shared-memory stage, and reaches 8 of its 9 rows and 256 of its 257 columns at the 2x step
    rows = cols = 0
    for c in ac.CASES:
        if c["geom"] != ac.GEOM_RESIZE:
            continue
        nbx, nby = ac.tile_grid(c)
        for by in range(nby):
            for bx in range(nbx):
                w = ac.stage_window(c, bx, by)
                if w:
                    rows, cols = max(rows, w[1] - w[0] + 1), max(cols, w[3] - w[2] + 1)
    assert rows == (ac.TILE_Y - 1) * ac.MAX_SCALE + 2 and cols == (ac.TILE_X - 1) * ac.MAX_SCALE + 2


# ---- sensitivity --------------------------------------------------------------------------------------------------------------------
def test_restatement_matches_fixture():
    fx = _fixture()
    for c in ac.CASES:
        d = float(np.abs(restate(c) - fx[c["id"]]).max())
        assert d <= ac.tol(c), (c["id"], d)


PERTURBATIONS = [
    ("window_top_short", dict(shrink="top")),
    ("window_bottom_short", dict(shrink="bottom")),
    ("window_left_short", dict(shrink="left")),
    ("window_right_short", dict(shrink="right")),
    ("lin_coord_unclamped", dict(clamp=False)),
    ("coordinate_in_float32", dict(f32_coord=True)),
    ("hue_wrap_ge", dict(ge_wrap=True)),
    ("tie_g_before_r", dict(g_first=True)),
    ("warp_round_half_away", dict(half_away=True)),
    ("u8_remap_truncates", dict(no_plus512=True)),
]


@pytest.mark.parametrize("name, kw", PERTURBATIONS, ids=[p[0] for p in PERTURBATIONS])
def test_perturbation_moves_a_case_beyond_tolerance(name, kw):
    fx = _fixture()
    moved = []
    for c in ac.CASES:
        if ("shrink" in kw or "clamp" in kw or "f32_coord" in kw) and c["geom"] != ac.GEOM_RESIZE:
            continue
        if ("half_away" in kw or "no_plus512" in kw) and c["geom"] == ac.GEOM_RESIZE:
            continue
        d = float(np.abs(restate(c, **kw) - fx[c["id"]]).max())
        if d > ac.tol(c):
            moved.append(c["id"])
    assert moved, name
    print(f"{name}: {len(moved)} cases beyond tolerance, e.g. {moved[:3]}")


def test_dropping_the_grey_branch_changes_nothing():
    """cv2's HSV->RGB takes r = g = b = v when s == 0, but its sector formula gives the same there (every table entry is v * 1): no input can
    tell the branch's removal apart, so it is pinned as an equivalence rather than by a sensitivity case."""
    for c in ac.CASES:
        if c["group"] == "colour" and ac.OP_HSV2RGB in c["ops"]:
            assert np.array_equal(restate(c, drop_s0=True), restate(c)), c["id"]


# ---- the 2x stage's refusal boundary ----------------------------------------------------------------------------------------------------
def _describe(H, W, crop_top, Ho, Wo):
    frame = np.zeros((H, W, 3), np.uint8)
    f = ta.DeferredFrame(frame, ta.GEOM_RESIZE, crop_top, ac.IDENTITY, 0, np.zeros(0, np.int32), np.zeros(0, np.float32), np.zeros(3), Ho, Wo,
                         ac.MEAN, ac.STD)
    return f.describe(frame.ctypes.data)


def test_refusal_boundary_of_the_2x_stage():
    r = ac.REFUSED
    Hc = r["H"] - r["crop_top"]
    Hr, Wr, sy, sx = ac.resize_geom(Hc, r["W"], r["Ho"])
    assert sy == 2.0 and Wr == 50 and sx > 2.0
    with pytest.raises(_lib.Vd3dError, match="shrinks"):
        _describe(r["H"], r["W"], r["crop_top"], r["Ho"], r["Wo"])
    # the exact 2x step on both axes is accepted (and pinned by the impulse_2x cases)
    _describe(576, 600, 0, 288, 400)
    assert any(ac.geometry(c)[3:] == (2.0, 2.0) for c in ac.CASES if c["geom"] == ac.GEOM_RESIZE)
