"""The constructed rotated-box cases of tests/rotated_cases.py are what they claim: every closed-form area against the float64 clipper of
oracle/torch_port.py and against a second, independent computation; the two box conventions describe one corner set; and the float32
restatements of the two device routines stay within the stated bounds and collect the candidate-point counts each family promises."""
import math
from fractions import Fraction

import numpy as np
import pytest
from scipy.spatial import ConvexHull

import rotated_cases as rc
import torch_port as tp

ALL = rc.all_cases()
IDS = [f"{k.family}-{k.name}" for k in ALL]


def test_every_family_is_present_at_every_centre():
    assert len({(k.family, k.name) for k in ALL}) == len(ALL)
    for f in rc.FAMILIES:
        assert {k.centre for k in rc.cases(f)} == set(rc.CENTRES), f


@pytest.mark.parametrize("k", ALL, ids=IDS)
def test_boxes_are_exact_in_float32_and_conventions_agree(k):
    for b in (k.a, k.b):
        x, kk = rc.to_xyxy(b), rc.to_kitti(b)
        assert [rc.f32(v) for v in x] == x and [rc.f32(v) for v in kk] == kk
        assert rc.xyxy_to_kitti(x) == kk                                   # round trip, exact
        cx, ck = sorted(rc.corners_xyxy(x)), sorted(rc.corners_kitti(kk))
        assert np.abs(np.array(cx) - np.array(ck)).max() <= 1e-12 * max(1.0, abs(b[0]), abs(b[1]))


@pytest.mark.parametrize("k", [k for k in ALL if k.family != "flat"], ids=[i for i, k in zip(IDS, ALL) if k.family != "flat"])
def test_closed_form_matches_clipper(k):
    clip = tp.rotated_overlap_bev(np.array(rc.to_xyxy(k.a)), np.array(rc.to_xyxy(k.b)))
    assert abs(clip - k.area) <= 1e-9 * max(k.area, 1e-3)


def test_octagon_formula_against_the_square_form_and_the_hull_of_its_vertices():
    for s, d in ((2.0, 0.5), (3.0, math.pi / 4), (1.0, 1e-3)):
        assert abs(rc.octagon_area(s, s, d) - 2 * s * s / (1 + math.sin(d) + math.cos(d))) < 1e-12 * s * s
    for w, h, d in ((4.0, 2.0, 0.3), (1.5, 3.5, 0.35), (4.0, 1.75, 0.6)):       # the eight crossings, from the edge lines, then their hull
        a, b, c, s, th = w / 2, h / 2, math.cos(d), math.sin(d), math.tan(d / 2)
        v = [(a, a * th), ((a - b * s) / c, b), (-b * th, b), (-a, (b - a * s) / c)]
        v += [(-x, -y) for x, y in v]
        assert len(ConvexHull(np.array(v)).vertices) == 8
        assert abs(ConvexHull(np.array(v)).volume - rc.octagon_area(w, h, d)) < 1e-12 * w * h


def aligned_area_exact(a, b):
    """Axis-aligned pairs in rational arithmetic."""
    xa, xb = [[Fraction(v) for v in rc.to_xyxy(x)[:4]] for x in (a, b)]
    w = min(xa[2], xb[2]) - max(xa[0], xb[0])
    h = min(xa[3], xb[3]) - max(xa[1], xb[1])
    return max(w, Fraction(0)) * max(h, Fraction(0))


def test_degenerate_axis_aligned_cases_in_rational_arithmetic():
    seen = 0
    for k in ALL:
        if k.family in ("edge", "disjoint", "identical", "flat") and k.a[4] == 0 and k.b[4] == 0 and min(k.a[2:4] + k.b[2:4]) >= 0:
            assert aligned_area_exact(k.a, k.b) == Fraction(k.area), k.name
            seen += 1
    assert seen >= 28


def test_disjoint_cases_are_apart_and_diamonds_share_their_bounding_boxes():
    for k in rc.cases("disjoint"):
        ca, cb = np.array(rc.corners_kitti(k.a)), np.array(rc.corners_kitti(k.b))
        gap = max(max((cb @ n).min() - (ca @ n).max(), (ca @ n).min() - (cb @ n).max())                 # separating axis over the edge normals
                  for t in (k.a[4], k.b[4]) for n in (np.array([math.cos(t), -math.sin(t)]), np.array([math.sin(t), math.cos(t)])))
        assert gap > 9e-4, k.name
        if k.name.startswith("diamonds"):
            xa, xb = rc.to_xyxy(k.a), rc.to_xyxy(k.b)
            assert xa[2] > xb[0] and xa[3] > xb[1]


@pytest.mark.parametrize("k", ALL, ids=IDS)
def test_restatements_hold_the_bounds_and_the_promised_point_counts(k):
    ro, n_ro = rc.rotated_overlap_f32(rc.to_xyxy(k.a), rc.to_xyxy(k.b))
    rb, n_rb = rc.rbox_inter_f32(rc.to_kitti(k.a), rc.to_kitti(k.b))
    assert abs(ro - k.area) <= rc.overlap_bound(k) / 2
    if rc.rbox_bound(k) is not None:
        assert abs(rb - k.area) <= rc.rbox_bound(k) / 2
    name = k.name.split("#")[0]
    if k.family == "disjoint":
        assert (ro, n_ro, rb) == (0.0, 0, 0.0) and n_rb < 3                # parallel edges may yield a stray crossing: still no area
    elif k.family == "contain":
        assert n_ro == 4 and n_rb == 4                                     # the inner box's corners, no crossing
    elif k.family in ("angle", "thin") or name in ("octagon", "diamond"):
        assert (n_ro, n_rb) == ((8, 8) if k.family != "thin" else (4, 4))  # proper crossings only
    elif k.family == "identical":
        assert n_ro == 8                                                   # eight corners within the margin, no strict crossing
    elif name == "over8":
        assert n_rb > 8 and n_ro == 16
        rb8, _ = rc.rbox_inter_f32(rc.to_kitti(k.a), rc.to_kitti(k.b), slots=8)
        assert abs(rb8 - k.area) > 2 * rc.OVER8_BOUND                      # eight slots would lose a vertex of the intersection


def test_many_points_reaches_sixteen_candidates_for_rotated_overlap():
    counts = [rc.rotated_overlap_f32(rc.to_xyxy(k.a), rc.to_xyxy(k.b))[1] for k in rc.cases("many_points")]
    assert max(counts) == 16 and sum(c > 8 for c in counts) >= 16
    assert sum(k.name.startswith("over8") for k in rc.cases("many_points")) == len(rc.OVER8)


def test_identical_boxes_lose_area_in_rbox_inter_away_from_angle_zero():
    """Not a bound but a record of the conditioning the bounded assertions stand on: with both corner sets equal, the inclusive corner test of
    rbox_inter compares dot products that differ only by rounding, so a rectangle against itself can come out as 0 or as half its area."""
    got = {k.name: rc.rbox_inter_f32(rc.to_kitti(k.a), rc.to_kitti(k.b))[0] / k.area for k in rc.cases("identical")}
    assert all(abs(v - 1) < 1e-6 for n, v in got.items() if n.startswith("angle_0.00"))
    assert min(got.values()) == 0.0 and all(-1e-6 < v < 1 + 1e-6 for v in got.values())
