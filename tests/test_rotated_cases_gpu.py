"""-m gpu: the two rotated-rectangle overlap kernels (csrc/rotated_overlap.cuh through ops/iou3d.py, csrc/kitti_eval.cu::rbox_inter through
kitti_eval.rotate_iou), the pairwise launch shapes, the 3-D IoU wrapper and the BEV NMS (mask and sweep kernels of csrc/iou3d.cu) on the
constructed cases of tests/rotated_cases.py, whose answers are exact.  The error tables are printed (pytest -rP shows them)."""
import numpy as np
import pytest
import torch

import rotated_cases as rc
from visualdet3d_b200 import _lib, kitti_eval
from visualdet3d_b200.ops import iou3d

pytestmark = pytest.mark.gpu


def dev(rows):
    return torch.tensor(np.array(rows, dtype=np.float64), dtype=torch.float32, device="cuda").contiguous()


def pair_results(ks):
    """Per case: overlap and IoU of rotated_overlap, and rbox_inter at the four criteria with box a as the first argument."""
    A, B = dev([rc.to_xyxy(k.a) for k in ks]), dev([rc.to_xyxy(k.b) for k in ks])
    ov, io = torch.zeros(len(ks), len(ks), device="cuda"), torch.zeros(len(ks), len(ks), device="cuda")
    iou3d.boxes_overlap_bev_gpu(A, B, ov)
    iou3d.boxes_iou_bev_gpu(A, B, io)
    KA, KB = dev([rc.to_kitti(k.a) for k in ks]), dev([rc.to_kitti(k.b) for k in ks])
    rb = {c: torch.diagonal(kitti_eval.rotate_iou(KB, KA, c)).cpu().numpy().astype(np.float64) for c in (-1, 0, 1, 2)}
    return torch.diagonal(ov).cpu().numpy().astype(np.float64), torch.diagonal(io).cpu().numpy().astype(np.float64), rb


def areas(k):
    return k.a[2] * k.a[3], k.b[2] * k.b[3]


@pytest.mark.parametrize("family", rc.FAMILIES)
def test_areas_against_exact(family):
    """Every family against its closed-form area.  rotated_overlap holds `overlap_bound` everywhere; rbox_inter holds `rbox_bound` where one
    exists.  Where none exists (identical rectangles away from angle 0, turns below 1e-3 rad, zero-width boxes) its result is decided by
    rounding, exactly as the evaluator it restates: those values are printed, not asserted."""
    ks = rc.cases(family)
    ov, io, rb = pair_results(ks)
    rows = {}
    for i, k in enumerate(ks):
        sa, sb = areas(k)
        union = sa + sb - k.area
        ro_ref, _ = rc.rotated_overlap_f32(rc.to_xyxy(k.a), rc.to_xyxy(k.b))
        rb_ref, _ = rc.rbox_inter_f32(rc.to_kitti(k.a), rc.to_kitti(k.b))
        r = rows.setdefault(k.centre, [0.0, 0.0, 0.0, 0.0])
        r[0], r[2] = max(r[0], abs(ov[i] - k.area)), max(r[2], abs(ov[i] - ro_ref))
        assert np.isfinite(ov[i]) and np.isfinite(io[i]), k.name
        assert abs(ov[i] - k.area) <= rc.overlap_bound(k), (k.name, ov[i], k.area)
        if family == "disjoint":
            assert ov[i] == 0.0 and io[i] == 0.0 and all(rb[c][i] == 0.0 for c in rb), k.name
        if family in rc.EXACT_FAMILIES:
            assert abs(io[i] - k.area / union) <= 2 * rc.overlap_bound(k) * (sa + sb) / union ** 2 + 1e-6, k.name
        if family in ("well", "contain", "disjoint"):
            assert abs(ov[i] - ro_ref) <= rc.tolerance(k) / 2 and abs(rb[2][i] - rb_ref) <= rc.tolerance(k) / 4, k.name
        bound = rc.rbox_bound(k)
        if bound is None:
            continue
        r[1], r[3] = max(r[1], abs(rb[2][i] - k.area)), max(r[3], abs(rb[2][i] - rb_ref))
        assert abs(rb[2][i] - k.area) <= bound, (k.name, rb[2][i], k.area)
        assert 0 <= rb[2][i] <= min(abs(sa), abs(sb)) * (1 + 1e-4) + bound, k.name
        if family in rc.EXACT_FAMILIES or family == "edge":
            for c, want in ((-1, k.area / union), (0, k.area / sa), (1, k.area / sb)):
                assert abs(rb[c][i] - want) <= 2 * bound * (sa + sb) / min(sa, sb, union) ** 2 + 1e-6, (k.name, c)
    print(f"\n{family}: max |device - exact| and |device - float32 restatement| (m^2) per centre, rbox columns over the bounded cases only")
    for c, r in rows.items():
        print(f"  centre {str(c):14s} rotated_overlap {r[0]:.3e} (restatement {r[2]:.3e})   rbox_inter {r[1]:.3e} (restatement {r[3]:.3e})")
    unbounded = [(k.name, rb[2][i], k.area) for i, k in enumerate(ks) if rc.rbox_bound(k) is None]
    for name, got, want in unbounded:
        print(f"  rbox_inter, no bound: {name:32s} device {got:12.6f} exact {want:10.6f}")


def test_flat_boxes_pin_todays_values():
    """What a 2-D detector's result file carries as its 3-D box, and zero-area boxes.  rotated_overlap finds no point in a box with
    negative sizes, so the placeholder against itself overlaps by 0 there and by its 1 m^2 in rbox_inter.  Criteria 0 and 1 of rotate_iou divide
    by the first or second area, as the evaluator they restate does: with a zero-area box and no intersection that is 0 / 0 = NaN today."""
    ks = {k.name.split("#")[0]: k for k in rc.cases("flat", centres=((3.0, -2.0),))}
    names = list(ks)
    ov, io, rb = pair_results([ks[n] for n in names])
    i = names.index("placeholder_twice")
    assert ov[i] == 0.0 and io[i] == 0.0 and abs(rb[2][i] - 1.0) < 2e-4 and abs(rb[-1][i] - 1.0) < 4e-4
    for n in ("placeholder_real", "real_placeholder"):
        assert all(rb[c][names.index(n)] == 0.0 for c in rb) and ov[names.index(n)] == 0.0
    j = names.index("zero_area_both")
    assert rb[2][j] == 0.0 and np.isnan(rb[0][j]) and np.isnan(rb[1][j]) and np.isnan(rb[-1][j])
    assert ov[j] == 0.0 and io[j] == 0.0                                   # rotated_iou clamps its denominator at 1e-8


def test_invariances():
    """No oracle needed: swapping the arguments (criteria 0 and 1 of rotate_iou swap with them), and one geometry written with ry + pi on both
    boxes, ry +- 2 pi, and sides swapped with ry + pi/2, agree within the bound."""
    ks = [k for f in ("well", "contain", "thin", "angle", "edge") for k in rc.cases(f)]
    ov, io, rb = pair_results(ks)
    sw = [k._replace(a=k.b, b=k.a) for k in ks]
    ov2, io2, rb2 = pair_results(sw)
    for i, k in enumerate(ks):
        b = 2 * rc.tolerance(k)
        sa, sb = areas(k)
        assert abs(ov[i] - ov2[i]) <= b and abs(rb[2][i] - rb2[2][i]) <= b, k.name
        assert abs(rb[0][i] - rb2[1][i]) <= b / sa + 1e-6 and abs(rb[1][i] - rb2[0][i]) <= b / sb + 1e-6, k.name
    ang = rc.cases("angle")
    ov, io, rb = pair_results(ang)
    for c in rc.CENTRES:
        idx = [i for i, k in enumerate(ang) if k.centre == c]
        assert len(idx) == len(rc.ANGLE_VARIANTS)
        spread_o, spread_r = np.ptp(ov[idx]), np.ptp(rb[2][idx])
        print(f"angle variants at {c}: spread rotated_overlap {spread_o:.3e}, rbox_inter {spread_r:.3e}")
        assert max(spread_o, spread_r) <= 2 * rc.tolerance(ang[idx[0]])


def test_more_than_eight_candidate_points_use_the_24_slots():
    """rbox_inter keeps room for 24 candidate points where the evaluator it restates keeps 8.  These pairs produce 9 or 10; with all of them the
    area is within OVER8_BOUND of the exact one, with the first 8 alone it is not (test_rotated_cases_cpu.py)."""
    ks = [k for k in rc.cases("many_points") if k.name.startswith("over8")]
    assert len(ks) == len(rc.OVER8)
    _, _, rb = pair_results(ks)
    for i, k in enumerate(ks):
        print(f"{k.name}: device {rb[2][i]:.6f} exact {k.area:.6f}")
        assert abs(rb[2][i] - k.area) <= rc.OVER8_BOUND, k.name


def contained_sets(M, N, c=(3.0, -2.0)):
    """M outer and N inner boxes about one centre, every inner box inside every outer one: overlap[i][j] is the inner box's area."""
    outer = [rc.box(*c, *[(6, 5), (8, 4), (5, 5)][i % 3], 0.4 + 0.1 * i) for i in range(M)]
    inner = [rc.box(*rc.place(c, 0.3 * j, 0.5, 0.25), *[(2, 1), (1.5, 1.5), (0.5, 2.5)][j % 3], -0.8 + 0.07 * j) for j in range(N)]
    return outer, inner


@pytest.mark.parametrize("M", [1, 15, 16, 17, 33])
@pytest.mark.parametrize("N", [1, 15, 16, 17, 33])
def test_pairwise_launch_shapes(M, N):
    """pairwise_kernel runs 16 x 16 blocks and rotate_iou_kernel 128 threads over M * N: sizes at and around the block edges, every element
    against its exact value and the 64 floats after the M * N outputs untouched."""
    outer, inner = contained_sets(M, N)
    want = np.array([[b[2] * b[3] for b in inner]] * M)
    A, B = dev([rc.to_xyxy(b) for b in outer]), dev([rc.to_xyxy(b) for b in inner])
    tol = rc.TOL_C * 2.0 ** -23 * (3 + 10) ** 2
    for fn, scale in ((iou3d.boxes_overlap_bev_gpu, 1.0), (iou3d.boxes_iou_bev_gpu, None)):
        buf = torch.full((M * N + 64,), -7.0, device="cuda")
        fn(A, B, buf[:M * N].view(M, N))
        got = buf.cpu().numpy()
        exp = want if scale else want / np.array([[o[2] * o[3]] for o in outer])       # IoU of a contained box: inner / outer
        assert np.abs(got[:M * N].reshape(M, N) - exp).max() <= tol and (got[M * N:] == -7.0).all()
    KA, KB = dev([rc.to_kitti(b) for b in outer]), dev([rc.to_kitti(b) for b in inner])
    buf = torch.full((M * N + 64,), -7.0, device="cuda")
    _lib.call("vd3d_kitti_rotate_iou", KA.data_ptr(), M, KB.data_ptr(), N, 2, buf.data_ptr(), torch.cuda.current_stream().cuda_stream)
    got = buf.cpu().numpy()
    assert np.abs(got[:M * N].reshape(M, N) - want).max() <= tol and (got[M * N:] == -7.0).all()


def test_pairwise_empty_sides_write_nothing():
    outer, inner = contained_sets(3, 3)
    A, B = dev([rc.to_xyxy(b) for b in outer]), dev([rc.to_xyxy(b) for b in inner])
    st = torch.cuda.current_stream().cuda_stream
    for M, N in ((0, 3), (3, 0), (0, 0)):
        buf = torch.full((64,), -7.0, device="cuda")
        for name in ("vd3d_boxes_overlap_bev", "vd3d_boxes_iou_bev"):
            _lib.call(name, A.data_ptr(), M, B.data_ptr(), N, buf.data_ptr(), st)
        _lib.call("vd3d_kitti_rotate_iou", A.data_ptr(), M, B.data_ptr(), N, -1, buf.data_ptr(), st)
        assert (buf.cpu().numpy() == -7.0).all()
    assert kitti_eval.rotate_iou(A[:0], B).shape == (0, 3)


def test_boxes_iou3d_closed_forms():
    """[x, y, z, h, w, l, ry] with the box spanning [y - h, y]: footprints from the constructed families, heights chosen by hand."""
    a = [1.0, 0.0, 10.0, 2.0, 1.5, 4.0, 0.3]
    half = [1.0, 1.0, 10.0, 2.0, 1.5, 4.0, 0.3]                          # same footprint, half the height shared: 1 / (2 + 2 - 1)
    above = [1.0, -2.5, 10.0, 2.0, 1.5, 4.0, 0.3]                        # same footprint, heights apart
    inner = [1.0, 0.0, 10.0, 2.0, 0.5, 1.0, 1.1]                         # footprint inside a's, same height span: 1 / 12
    inner_above = [1.0, 3.0, 10.0, 2.0, 0.5, 1.0, 1.1]
    A, B = dev([a]), dev([a, half, above, inner, inner_above])
    got = iou3d.boxes_iou3d_gpu(A, B).cpu().numpy()[0]
    assert np.abs(got - np.array([1.0, 1 / 3, 0.0, 1 / 12, 0.0])).max() <= 1e-5
    assert got[2] == 0.0 and got[4] == 0.0
    assert np.abs(iou3d.boxes_iou3d_gpu(B, A).cpu().numpy()[:, 0] - got).max() <= 1e-5


# ---- NMS: axis-aligned boxes on a 0.5 m grid, so every IoU is exact in float32 and in the float64 host sweep alike --------------------
def row_boxes(xs, w=4.0, h=2.0):
    xs = np.asarray(xs, dtype=np.float64)
    return np.stack([xs - w / 2, np.full_like(xs, -h / 2), xs + w / 2, np.full_like(xs, h / 2), np.zeros_like(xs)], 1)


def exact_iou(b):
    w = np.clip(np.minimum(b[:, None, 2], b[None, :, 2]) - np.maximum(b[:, None, 0], b[None, :, 0]), 0, None)
    h = np.clip(np.minimum(b[:, None, 3], b[None, :, 3]) - np.maximum(b[:, None, 1], b[None, :, 1]), 0, None)
    s = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    return w * h / (s[:, None] + s[None, :] - w * h)


def host_nms(b, thr, at_threshold=False):
    iou = exact_iou(b)
    assert at_threshold or np.abs(iou - thr).min() > 1e-4                   # no decision rests on rounding unless the case says so
    alive, keep = np.ones(len(b), bool), []
    for i in range(len(b)):
        if alive[i]:
            keep.append(i)
            alive[i + 1:] &= ~(iou[i, i + 1:] > thr)
    return keep


def run_nms(fn, b, thr):
    keep = torch.full((len(b),), -1, dtype=torch.int64)
    n = fn(dev(b), keep, thr)
    assert (keep[n:] == -1).all()                                           # nothing written beyond the returned count
    return keep[:n].tolist()


def grouped(n):
    """Groups of four 4 x 2 boxes shifted by 0, 1, 2, 3 m (IoU 3/5, 1/3, 1/7 by distance), groups 8 m apart.  At 0.5: box 0 suppresses box 1,
    box 2 overlaps only box 1 above the threshold and so stays, and suppresses box 3."""
    i = np.arange(n)
    return row_boxes(8.0 * (i // 4) + (i % 4))


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 127, 128, 129, 2047, 2048, 2049, 4100])
def test_nms_sizes_around_the_mask_words(n):
    """n up to 4100 is 65 mask words per row: the sweep's 32 lanes each take more than one word.  Box 2565 (word 40) repeats box 0 and must go.
    Box 2630 (word 41) is box 65 moved 0.5 m sideways: above the threshold only against box 65 (word 1), which box 64 has already
    suppressed, so it must stay."""
    b = grouped(n)
    if n > 2630:
        b[2565], b[2630] = b[0], b[65] + np.array([0, 0.5, 0, 0.5, 0])
    want = host_nms(b, 0.5)
    assert (n <= 2630) or (2565 not in want and 2630 in want)
    for fn in (iou3d.nms_gpu, iou3d.nms_normal_gpu):
        assert run_nms(fn, b, 0.5) == want


@pytest.mark.parametrize("n", [65, 130, 2050])
def test_nms_chain_across_word_boundaries(n):
    """Boxes 1 m apart: each suppresses only its successor, so the even indices stay; pairs (63, 64) and (2047, 2048) straddle mask words."""
    b = row_boxes(np.arange(n, dtype=np.float64))
    want = host_nms(b, 0.5)
    assert want == list(range(0, n, 2))
    for fn in (iou3d.nms_gpu, iou3d.nms_normal_gpu):
        assert run_nms(fn, b, 0.5) == want


@pytest.mark.parametrize("n", [64, 200])
def test_nms_all_identical_and_all_disjoint(n):
    for fn in (iou3d.nms_gpu, iou3d.nms_normal_gpu):
        assert run_nms(fn, row_boxes(np.zeros(n)), 0.5) == [0]
        assert run_nms(fn, row_boxes(8.0 * np.arange(n)), 0.5) == list(range(n))


def test_nms_iou_exactly_at_the_threshold_is_kept():
    """IoU 4 / 12 and 4 / 8 are computed without rounding beyond the final quotient, so the strict `>` is decidable through the axis-aligned
    branch: at the threshold the box stays, one float32 step below it goes.  The rotated branch is held to thresholds 1e-3 either side."""
    third = row_boxes([0.0, 2.0])                                          # 4 x 2, shifted 2: 4 / 12
    half = row_boxes([0.0, 1.0], w=3.0)                                    # 3 x 2, shifted 1: 4 / 8
    for b, v in ((third, np.float32(1) / np.float32(3)), (half, np.float32(0.5))):
        assert abs(exact_iou(b)[0, 1] - float(v)) < 1e-7
        assert run_nms(iou3d.nms_normal_gpu, b, float(v)) == [0, 1]
        assert run_nms(iou3d.nms_normal_gpu, b, float(np.nextafter(v, np.float32(0)))) == [0]
        assert run_nms(iou3d.nms_gpu, b, float(v) + 1e-3) == [0, 1]
        assert run_nms(iou3d.nms_gpu, b, float(v) - 1e-3) == [0]


def test_nms_mask_holds_later_boxes_only():
    """The suppression mask itself, from a row's own 64-box word on (the sweep reads no earlier word): bit j of row i is set exactly when j > i
    and IoU(i, j) > threshold, so a box never marks itself or an earlier box of its word.  The last, partial word carries no bit at or beyond n."""
    n = 130
    b = row_boxes(np.arange(n, dtype=np.float64))
    boxes = dev(b)
    words = (n + 63) // 64
    ws = torch.zeros(int(_lib.load().vd3d_nms_bev_workspace(n)), dtype=torch.uint8, device="cuda")
    keep, count = torch.empty(n, dtype=torch.int64, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    want = np.triu(exact_iou(b) > 0.5, 1)
    read = np.arange(words * 64)[None, :] // 64 >= np.arange(n)[:, None] // 64
    for rotated in (1, 0):
        _lib.call("vd3d_nms_bev", boxes.data_ptr(), n, 0.5, rotated, ws.data_ptr(), keep.data_ptr(), count.data_ptr(),
                  torch.cuda.current_stream().cuda_stream)
        mask = ws.cpu().numpy()[:n * words * 8].view(np.uint64).reshape(n, words)
        bits = ((mask[:, :, None] >> np.arange(64, dtype=np.uint64)) & np.uint64(1)).astype(bool).reshape(n, words * 64)
        assert np.array_equal((bits & read)[:, :n], want) and not bits[:, n:].any()
        assert int(count.item()) == n // 2


def test_nms_refuses_more_boxes_than_the_sweep_can_hold():
    """The sweep keeps one 64-bit word per 64 boxes in 48 KB of shared memory; beyond that the entry refuses before any launch."""
    small = torch.zeros(64, device="cuda")
    keep, count = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.Vd3dError, match="too many boxes"):
        _lib.call("vd3d_nms_bev", small.data_ptr(), 48 * 1024 * 8 + 1, 0.5, 1, small.data_ptr(), keep.data_ptr(), count.data_ptr(),
                  torch.cuda.current_stream().cuda_stream)
