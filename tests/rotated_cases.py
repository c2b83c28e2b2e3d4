"""Constructed rotated-rectangle pairs whose intersection area is known in closed form (float64, no clipper involved), for the two
float32 overlap routines of the library, plus a float32 numpy restatement of each routine.

Conventions.  csrc/rotated_overlap.cuh takes [x1, y1, x2, y2, ry]; csrc/kitti_eval.cu::rbox_inter takes [cx, cy, dx, dy, angle].  Both place
a corner with local offset (lx, ly) at centre + (lx cos t + ly sin t, -lx sin t + ly cos t), so one box (cx, cy, w, h, t) is
[cx - w/2, cy - h/2, cx + w/2, cy + h/2, t] for the first and [cx, cy, w, h, t] for the second (`to_xyxy`, `to_kitti`; proved on the corner
sets in test_rotated_cases_cpu.py).  Every builder snaps centres to a 1/1024 m grid, sizes to 1/512 m and angles to float32, so both forms are
exact in float32, and computes the area from the snapped values.

Families (`FAMILIES`): well, contain, disjoint, identical, edge, angle, thin, many_points, flat; each at the centres `CENTRES` (the last two
are KITTI range).  `cases(family)` lists them.

The restatements (`rotated_overlap_f32`, `rbox_inter_f32`) follow the device code operation for operation in np.float32.  They are not
oracles: they tell, without a GPU, which constructed cases are well conditioned in float32, how many candidate points a case produces and what
error to expect.  rbox_inter is compiled without FMA contraction and takes cos / sin in double, so its restatement is expected to agree with
the device to the last bits; rotated_overlap is compiled with contraction and uses cosf / sinf / atan2f, so its restatement agrees to a few ulp.
"""
import math
from collections import namedtuple

import numpy as np

CENTRES = ((0.0, 0.0), (3.0, -2.0), (-25.0, 45.0), (40.0, 78.0))
FAMILIES = ("well", "contain", "disjoint", "identical", "edge", "angle", "thin", "many_points", "flat")
EXACT_FAMILIES = ("well", "contain", "identical", "angle", "thin")        # held to the derived tolerance `tolerance(case)`
BOUNDED_FAMILIES = ("edge", "many_points", "flat")                         # held to bounded statements only
TOL_C = 4.0                                                               # the one constant of `tolerance`

Case = namedtuple("Case", "family name centre a b area")                   # a, b: (cx, cy, w, h, t) float64, float32-representable


def f32(v):
    return float(np.float32(v))


def box(cx, cy, w, h, t):
    return (round(cx * 1024) / 1024, round(cy * 1024) / 1024, round(w * 512) / 512, round(h * 512) / 512, f32(t))


def to_xyxy(b):
    cx, cy, w, h, t = b
    return [cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, t]


def to_kitti(b):
    return list(b)


def xyxy_to_kitti(x):
    return [(x[0] + x[2]) / 2, (x[1] + x[3]) / 2, x[2] - x[0], x[3] - x[1], x[4]]


def corners_xyxy(x):
    """rotated_corners of rotated_overlap.cuh in float64."""
    x1, y1, x2, y2, t = x
    cx, cy, c, s = (x1 + x2) / 2, (y1 + y2) / 2, math.cos(t), math.sin(t)
    return [((px - cx) * c + (py - cy) * s + cx, -(px - cx) * s + (py - cy) * c + cy) for px, py in ((x1, y1), (x2, y1), (x2, y2), (x1, y2))]


def corners_kitti(k):
    """rbox_corners of kitti_eval.cu in float64."""
    c, s, hx, hy = math.cos(k[4]), math.sin(k[4]), k[2] / 2, k[3] / 2
    return [(c * lx + s * ly + k[0], -s * lx + c * ly + k[1]) for lx, ly in ((-hx, -hy), (-hx, hy), (hx, hy), (hx, -hy))]


def place(c, t, lx, ly):
    """World position of the local offset (lx, ly) of a box centred at c with angle t."""
    return (c[0] + lx * math.cos(t) + ly * math.sin(t), c[1] - lx * math.sin(t) + ly * math.cos(t))


def local(b, p):
    """Offset of the world point p in the frame of box b."""
    dx, dy, c, s = p[0] - b[0], p[1] - b[1], math.cos(b[4]), math.sin(b[4])
    return (dx * c - dy * s, dx * s + dy * c)


def diag(b):
    return math.hypot(b[2], b[3])


def tolerance(case):
    """Absolute float32 error allowed on the area of an EXACT_FAMILIES case: corner coordinates carry an error of about one ulp of
    (|centre| + diagonal), and the area is a sum of products of two of them."""
    reach = max(abs(case.centre[0]), abs(case.centre[1])) + max(diag(case.a), diag(case.b))
    return TOL_C * 2.0 ** -23 * reach * reach


# ---- closed forms --------------------------------------------------------------------------------------------------------------------
def octagon_area(w, h, d):
    """Two equal w x h rectangles about one centre, one turned by d against the other: the rectangle minus the four corner triangles the
    other's edges cut off.  Valid while every corner is cut by exactly one edge: 0 < tan(d/2) < min(w/h, h/w) after reducing d to (-pi/2, pi/2]."""
    d = abs((d + math.pi / 2) % math.pi - math.pi / 2)
    if d == 0:
        return w * h
    a, b, c, s, th = w / 2, h / 2, math.cos(d), math.sin(d), math.tan(d / 2)
    assert th < min(a / b, b / a), "octagon_area: angle too large for this aspect"
    t1 = (b - a * th) * (a * c - a + b * s) / c / 2
    t2 = (a - b * th) * (b * c - b + a * s) / c / 2
    return 4 * a * b - 2 * t1 - 2 * t2


def diamond_in_box_area(wa, ha, s):
    """An s x s square at 45 degrees against a concentric axis-aligned wa x ha rectangle that cuts all four of its tips and none of its edges whole."""
    r, a, b = s / math.sqrt(2), wa / 2, ha / 2
    assert a < r and b < r and a + b > r
    return 2 * r * r - 2 * (r - a) ** 2 - 2 * (r - b) ** 2


def shifted_area(a, b):
    """Equal angles: the overlap of the two extents along each local axis."""
    lx, ly = local(a, (b[0], b[1]))
    ox = min(a[2] / 2, lx + b[2] / 2) - max(-a[2] / 2, lx - b[2] / 2)
    oy = min(a[3] / 2, ly + b[3] / 2) - max(-a[3] / 2, ly - b[3] / 2)
    return max(ox, 0.0) * max(oy, 0.0)


# ---- families -------------------------------------------------------------------------------------------------------------------------
def _well(c):
    out = []
    for w, h, t0, d in ((2, 2, 0.0, 0.5), (3, 3, 0.7, math.pi / 4), (4, 2, -1.1, 0.3), (1.5, 3.5, 2.0, -0.35), (4, 1.75, 0.0, 0.6)):
        a, b = box(*c, w, h, t0), box(*c, w, h, t0 + d)
        out.append(("octagon", a, b, octagon_area(a[2], a[3], b[4] - a[4])))
    for wa, ha, s in ((2.5, 2.0, 2.5), (4.0, 3.0, 4.5)):
        a, b = box(*c, wa, ha, 0.0), box(*c, s, s, math.pi / 4)
        out.append(("diamond", a, b, diamond_in_box_area(a[2], a[3], b[2])))
    for w, h, dx, dy, t0 in ((4, 1.75, 1.0, 0.0, 0.0), (4, 1.75, 1.25, 0.0, 0.9), (2, 3, 0.0, 1.5, -2.3), (3.9, 1.6, 1.1, 0.4, 1.3)):
        a = box(*c, w, h, t0)
        b = box(*place(c, a[4], dx, dy), w, h, t0)
        out.append(("shift", a, b, shifted_area(a, b)))
    return out


def _contain(c):
    out = []
    for (W, H, t0), (w, h, t1), (ox, oy) in (((6, 5, 0.0), (2, 1, 0.0), (0.5, -0.25)), ((6, 5, 0.4), (2, 1, 1.7), (-0.5, 0.5)),
                                             ((8, 4, -2.0), (1.5, 1.5, 0.3), (0.5, 0.0)), ((5, 5, 3.0), (0.5, 3, -0.8), (0.0, 0.0))):
        a = box(*c, W, H, t0)
        b = box(*place(c, a[4], ox, oy), w, h, t1)
        assert math.hypot(ox, oy) + diag(b) / 2 < min(W, H) / 2 - 0.01
        out += [("inner_second", a, b, b[2] * b[3]), ("inner_first", b, a, b[2] * b[3])]
    return out


def _disjoint(c):
    out = []
    for gap in (1 / 1024, 1.0, 50.0):
        out.append((f"aligned_gap_{gap:g}", box(*c, 3, 2, 0.0), box(c[0] + 3 + gap, c[1], 3, 2, 0.0), 0.0))
    for gap in (1 / 256, 1.0):
        a = box(*c, 3, 2, 0.6)
        b = box(*place(c, a[4], 3 + gap, 0.25), 3, 2, 0.6)
        lx, _ = local(a, (b[0], b[1]))
        assert lx - 3 > 1 / 1024
        out.append((f"rotated_gap_{gap:g}", a, b, 0.0))
    for off in (1.5, math.sqrt(2) + 3 / 1024):          # two 2 x 2 diamonds corner to corner: tips r = sqrt(2) apart along the diagonal
        a, b = box(*c, 2, 2, math.pi / 4), box(c[0] + off, c[1] + off, 2, 2, math.pi / 4)
        assert math.sqrt(2) + 1 / 1024 < b[0] - a[0] < 2 * math.sqrt(2)      # apart, yet the axis-aligned boxes [x1, x2] overlap
        out.append((f"diamonds_{off:.3f}", a, b, 0.0))
    return out


def _identical(c):
    return [(f"angle_{t:.2f}", box(*c, 3.9, 1.6, t), box(*c, 3.9, 1.6, t), box(*c, 3.9, 1.6, t)[2] * box(*c, 3.9, 1.6, t)[3])
            for t in (0.0, 0.3, math.pi / 2, -math.pi, 3.0)]


def _edge(c):
    out = []
    a = box(*c, 4, 2, 0.0)
    out.append(("full_edge", a, box(c[0] + 4, c[1], 4, 2, 0.0), 0.0))
    out.append(("partial_edge", a, box(c[0] + 4, c[1] + 1, 4, 2, 0.0), 0.0))
    out.append(("collinear_shift", a, box(c[0] + 1, c[1], 4, 2, 0.0), 6.0))
    out.append(("vertex_on_vertex", a, box(c[0] + 4, c[1] + 2, 4, 2, 0.0), 0.0))
    ar = box(*c, 4, 2, 0.3)                              # the same, turned: the shared edge is no longer on a coordinate line
    out.append(("full_edge_turned", ar, box(*place(c, ar[4], 4, 0), 4, 2, 0.3), None))
    out.append(("collinear_shift_turned", ar, box(*place(c, ar[4], 1, 0), 4, 2, 0.3), None))
    for name, s in (("vertex_on_edge_outside", 1), ("vertex_on_edge_inside", -1)):
        r = 1 / math.sqrt(2)                             # a 1 x 1 diamond whose tip touches a's right edge from either side
        b = box(c[0] + 2 + s * r, c[1], 1, 1, math.pi / 4)
        dip = (a[0] + 2) - (b[0] - r) if s > 0 else (b[0] + r) - (a[0] + 2)      # how far the tip crosses the edge after snapping the centre
        out.append((name, a, b, max(dip, 0.0) ** 2 if s > 0 else 1.0 - max(dip, 0.0) ** 2))
    return [(n, x, y, shifted_area(x, y) if ar_ is None else ar_) for n, x, y, ar_ in out]


ANGLE_VARIANTS = ("base", "both_plus_pi", "plus_2pi", "minus_2pi", "swap_first", "swap_second", "swap_both")


def _angle(c):
    """One geometry (a 4 x 2 rectangle at 0.4 and at 0.9 about one centre) written seven ways; the area is recomputed from each variant's own
    float32 angles."""
    w, h, ta, tb = 4.0, 2.0, 0.4, 0.9
    forms = {"base": ((w, h, ta), (w, h, tb)), "both_plus_pi": ((w, h, ta + math.pi), (w, h, tb + math.pi)),
             "plus_2pi": ((w, h, ta + 2 * math.pi), (w, h, tb + 2 * math.pi)), "minus_2pi": ((w, h, ta - 2 * math.pi), (w, h, tb - 2 * math.pi)),
             "swap_first": ((h, w, ta + math.pi / 2), (w, h, tb)), "swap_second": ((w, h, ta), (h, w, tb + math.pi / 2)),
             "swap_both": ((h, w, ta + math.pi / 2), (h, w, tb + math.pi / 2))}
    out = []
    for name in ANGLE_VARIANTS:
        a, b = (box(*c, *f) for f in forms[name])
        ea = a[4] - (math.pi / 2 if name in ("swap_first", "swap_both") else 0)      # the angle of the 4 m axis
        eb = b[4] - (math.pi / 2 if name in ("swap_second", "swap_both") else 0)
        out.append((name, a, b, octagon_area(w, h, eb - ea)))
    return out


def _thin(c):
    out = []
    for t0, d in ((0.0, 0.0), (0.0, 0.2), (0.5, 0.7), (-1.2, 1.0), (2.5, -0.4)):
        a, b = box(*c, 4, 1.8, t0), box(*c, 26 / 512, 2600 / 512, t0 + d)             # 100 : 1, its long axis at d to a's short one
        dd = b[4] - a[4]
        assert a[3] / 2 * abs(math.tan(dd)) + b[2] / 2 / math.cos(dd) < a[2] / 2
        assert a[3] / 2 / math.cos(dd) + b[2] / 2 * abs(math.tan(dd)) < b[3] / 2
        out.append((f"strip_{d:g}", a, b, b[2] * a[3] / math.cos(dd)))
    return out


# (centre, w, h, angle, turn): pairs one or two float32 steps of the angle apart, found by running `rbox_inter_f32` over random draws, for
# which rbox_inter collects 9 or 10 candidate points, its 24-slot result is within OVER8_BOUND of the exact area and the first 8 alone are not.
OVER8 = (((0.0, 0.0), 3.9, 1.6, -3.06, 3.9e-07), ((0.0, 0.0), 4, 2, 1.7, 5.8e-07), ((0.0, 0.0), 4, 1.75, 0.43, 4e-07),
         ((0.0, 0.0), 4, 2, 1.11, 3.4e-07), ((0.0, 0.0), 3.9, 1.6, 2.58, 3.4e-07))
OVER8_BOUND = 5e-3


def _many_points(c):
    """Near-identical pairs: a rectangle against itself turned by a small angle about the common centre.  Exactly, all eight corners lie
    outside the other rectangle by about (half side) x angle and the edges cross eight times; in float32 corners within rounding (rbox_inter's
    inclusive test) or within 1e-5 m (rotated_overlap's margin) count as inside as well, so more than eight candidate points appear."""
    out = []
    for w, h, t0, d in ((4, 2, 0.3, 1e-2), (4, 2, 0.3, 1e-3), (3.9, 1.6, -1.0, 1e-5), (2, 2, 0.7, 4e-6), (4, 1.75, 2.0, 2e-6),
                        (2, 2, 0.0, 1e-6), (3, 1, 1.2, 3e-6)):
        a, b = box(*c, w, h, t0), box(*c, w, h, t0 + d)
        out.append((f"turn_{d:g}", a, b, octagon_area(a[2], a[3], b[4] - a[4])))
    for oc, w, h, t0, d in OVER8:
        if oc == c:
            a, b = box(*c, w, h, t0), box(*c, w, h, t0 + d)
            out.append(("over8", a, b, octagon_area(a[2], a[3], b[4] - a[4])))
    return out


def rbox_bound(case):
    """Absolute bound on |rbox_inter - exact area| that the restatement shows to hold for a BOUNDED_FAMILIES or `identical` case, or None where
    the routine's own conditioning allows none: its inclusive corner test and its crossing point (a quotient whose denominator vanishes for
    parallel edges) are decided by rounding once the two rectangles agree to within float32 resolution."""
    name = case.name.split("#")[0]
    if case.family == "edge":
        return tolerance(case)
    if case.family == "identical":
        return tolerance(case) if name == "angle_0.00" else None
    if case.family == "many_points":
        return {"turn_0.01": 8 * tolerance(case), "turn_0.001": 8 * tolerance(case) + 1e-3, "over8": OVER8_BOUND}.get(name)
    if case.family == "flat":
        return 2e-4 if name.startswith("placeholder") or name == "real_placeholder" else None
    return tolerance(case)


def overlap_bound(case):
    """The same for rotated_overlap, whose 1e-5 m margin and strict crossing keep every constructed case bounded; it finds no point in a box
    with negative sizes, so the placeholder against itself gives 0."""
    if case.family == "many_points":
        return 1e-4 + tolerance(case)
    if case.family == "flat" and case.name.startswith("placeholder_twice"):
        return 2.0
    return tolerance(case)


PLACEHOLDER = (-1000.0, -1000.0, -1.0, -1.0, f32(-10.0))      # what a 2-D detector's KITTI result file carries as its 3-D box


def _flat(c):
    real = box(*c, 4, 2, 0.3)
    return [("zero_width", box(*c, 0, 2, 0.0), real, 0.0), ("zero_width_turned", real, box(*c, 0, 2, 1.0), 0.0),
            ("zero_area", box(*c, 0, 0, 0.0), real, 0.0), ("zero_area_both", box(*c, 0, 0, 0.0), box(*c, 0, 0, 0.5), 0.0),
            ("placeholder_real", PLACEHOLDER, real, 0.0), ("real_placeholder", real, PLACEHOLDER, 0.0),
            ("placeholder_twice", PLACEHOLDER, PLACEHOLDER, 1.0)]      # the same corner set as a 1 x 1 box, walked the other way


_BUILDERS = dict(well=_well, contain=_contain, disjoint=_disjoint, identical=_identical, edge=_edge, angle=_angle, thin=_thin,
                 many_points=_many_points, flat=_flat)


def cases(family, centres=CENTRES):
    return [Case(family, f"{name}#{i}@{c[0]:g},{c[1]:g}", c, a, b, float(area)) for c in centres
            for i, (name, a, b, area) in enumerate(_BUILDERS[family](c))]


def all_cases():
    return [k for f in FAMILIES for k in cases(f)]


# ---- float32 restatements of the two device routines ----------------------------------------------------------------------------------
F = np.float32


def rotated_overlap_f32(a, b):
    """rotated_overlap of csrc/rotated_overlap.cuh on [x1, y1, x2, y2, ry] boxes -> (area, candidate points)."""
    a, b = [F(v) for v in a], [F(v) for v in b]
    two, eps, margin = F(2), F(1e-8), F(1e-5)

    def corners(bx):
        x1, y1, x2, y2, t = bx
        cx, cy, ac, as_ = (x1 + x2) / two, (y1 + y2) / two, np.cos(t), np.sin(t)
        c = [((px - cx) * ac + (py - cy) * as_ + cx, -(px - cx) * as_ + (py - cy) * ac + cy) for px, py in ((x1, y1), (x2, y1), (x2, y2), (x1, y2))]
        return c + [c[0]]

    def cross3(p1, p2, p0):
        return (p1[0] - p0[0]) * (p2[1] - p0[1]) - (p2[0] - p0[0]) * (p1[1] - p0[1])

    def seg(p1, p0, q1, q0):
        if not (min(p0[0], p1[0]) <= max(q0[0], q1[0]) and min(q0[0], q1[0]) <= max(p0[0], p1[0]) and
                min(p0[1], p1[1]) <= max(q0[1], q1[1]) and min(q0[1], q1[1]) <= max(p0[1], p1[1])):
            return None
        s1, s2, s3, s4 = cross3(q0, p1, p0), cross3(p1, q1, p0), cross3(p0, q1, q0), cross3(q1, p1, q0)
        if not (s1 * s2 > 0 and s3 * s4 > 0):
            return None
        s5 = cross3(q1, p1, p0)
        if abs(s5 - s1) > eps:
            return ((s5 * q0[0] - s1 * q1[0]) / (s5 - s1), (s5 * q0[1] - s1 * q1[1]) / (s5 - s1))
        a0, b0, c0 = p0[1] - p1[1], p1[0] - p0[0], p0[0] * p1[1] - p1[0] * p0[1]
        a1, b1, c1 = q0[1] - q1[1], q1[0] - q0[0], q0[0] * q1[1] - q1[0] * q0[1]
        D = a0 * b1 - a1 * b0
        return ((b0 * c1 - b1 * c0) / D, (a1 * c0 - a0 * c1) / D)

    def inside(bx, p):
        cx, cy, ac, as_ = (bx[0] + bx[2]) / two, (bx[1] + bx[3]) / two, np.cos(-bx[4]), np.sin(-bx[4])
        rx = (p[0] - cx) * ac + (p[1] - cy) * as_ + cx
        ry = -(p[0] - cx) * as_ + (p[1] - cy) * ac + cy
        return rx > bx[0] - margin and rx < bx[2] + margin and ry > bx[1] - margin and ry < bx[3] + margin

    with np.errstate(all="ignore"):
        ca, cb = corners(a), corners(b)
        pts = []
        for i in range(4):
            for j in range(4):
                x = seg(ca[i + 1], ca[i], cb[j + 1], cb[j])
                if x is not None:
                    pts.append(x)
        for k in range(4):
            if inside(a, cb[k]):
                pts.append(cb[k])
            if inside(b, ca[k]):
                pts.append(ca[k])
        n = len(pts)
        if n == 0:
            return 0.0, 0
        sx = sy = F(0)
        for p in pts:
            sx, sy = sx + p[0], sy + p[1]
        mx, my = sx / F(n), sy / F(n)
        ang = [np.arctan2(p[1] - my, p[0] - mx) for p in pts]
        for j in range(n - 1):
            for i in range(n - j - 1):
                if ang[i] > ang[i + 1]:
                    ang[i], ang[i + 1] = ang[i + 1], ang[i]
                    pts[i], pts[i + 1] = pts[i + 1], pts[i]
        area = F(0)
        for k in range(n - 1):
            ax, ay = pts[k][0] - pts[0][0], pts[k][1] - pts[0][1]
            bx, by = pts[k + 1][0] - pts[0][0], pts[k + 1][1] - pts[0][1]
            area = area + (ax * by - ay * bx)
        return float(abs(area) / two), n


def rbox_inter_f32(b1, b2, slots=24):
    """rbox_inter of csrc/kitti_eval.cu on [cx, cy, dx, dy, angle] boxes -> (area, candidate points found).  `slots` is the room for candidate
    points: 24 in the library; with 8 (the size of the buffer the evaluator was modelled on) later candidates are dropped here."""
    b1, b2 = [F(v) for v in b1], [F(v) for v in b2]
    two = F(2)

    def corners(b):
        ac, as_ = F(math.cos(float(b[4]))), F(math.sin(float(b[4])))
        hx, hy, px, py = -b[2] / two, -b[3] / two, b[2] / two, b[3] / two
        c = []
        for x, y in ((hx, hy), (hx, py), (px, py), (px, hy)):
            c += [ac * x + as_ * y + b[0], -as_ * x + ac * y + b[1]]
        return c

    def in_quad(x, y, c):
        ab0, ab1, ad0, ad1 = c[2] - c[0], c[3] - c[1], c[6] - c[0], c[7] - c[1]
        ap0, ap1 = x - c[0], y - c[1]
        abab, abap = ab0 * ab0 + ab1 * ab1, ab0 * ap0 + ab1 * ap1
        adad, adap = ad0 * ad0 + ad1 * ad1, ad0 * ap0 + ad1 * ap1
        return abab >= abap and abap >= 0 and adad >= adap and adap >= 0

    def seg(p1, p2, i, j):
        A0, A1, B0, B1 = p1[2 * i], p1[2 * i + 1], p1[2 * ((i + 1) % 4)], p1[2 * ((i + 1) % 4) + 1]
        C0, C1, D0, D1 = p2[2 * j], p2[2 * j + 1], p2[2 * ((j + 1) % 4)], p2[2 * ((j + 1) % 4) + 1]
        BA0, BA1, DA0, CA0, DA1, CA1 = B0 - A0, B1 - A1, D0 - A0, C0 - A0, D1 - A1, C1 - A1
        acd = DA1 * CA0 > CA1 * DA0
        bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0)
        if acd != bcd:
            abc = CA1 * BA0 > BA1 * CA0
            abd = DA1 * BA0 > BA1 * DA0
            if abc != abd:
                DC0, DC1 = D0 - C0, D1 - C1
                ABBA, CDDC = A0 * B1 - B0 * A1, C0 * D1 - D0 * C1
                DH = BA1 * DC0 - BA0 * DC1
                return ((ABBA * DC0 - BA0 * CDDC) / DH, (ABBA * DC1 - BA1 * CDDC) / DH)
        return None

    with np.errstate(all="ignore"):
        c1, c2 = corners(b1), corners(b2)
        p = []
        for i in range(4):
            if in_quad(c1[2 * i], c1[2 * i + 1], c2):
                p.append((c1[2 * i], c1[2 * i + 1]))
            if in_quad(c2[2 * i], c2[2 * i + 1], c1):
                p.append((c2[2 * i], c2[2 * i + 1]))
        for i in range(4):
            for j in range(4):
                t = seg(c1, c2, i, j)
                if t is not None:
                    p.append(t)
        found = len(p)
        p = p[:slots]
        n = len(p)
        if n > 0:
            cx = cy = F(0)
            for q in p:
                cx, cy = cx + q[0], cy + q[1]
            cx, cy = cx / F(n), cy / F(n)
            vs = []
            for q in p:
                v0, v1 = q[0] - cx, q[1] - cy
                d = np.sqrt(v0 * v0 + v1 * v1)
                v0, v1 = v0 / d, v1 / d
                vs.append(F(-2) - v0 if v1 < 0 else v0)
            for i in range(1, n):
                if vs[i - 1] > vs[i]:
                    temp, tq, j = vs[i], p[i], i
                    while j > 0 and vs[j - 1] > temp:
                        vs[j], p[j] = vs[j - 1], p[j - 1]
                        j -= 1
                    vs[j], p[j] = temp, tq
        area = F(0)
        for i in range(n - 2):
            (ax, ay), (bx, by), (qx, qy) = p[0], p[i + 1], p[i + 2]
            area = area + abs(((ax - qx) * (by - qy) - (ay - qy) * (bx - qx)) / two)
        return float(area), found
