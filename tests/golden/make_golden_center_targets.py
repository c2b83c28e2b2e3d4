"""Golden vectors for visualdet3d_b200/center_targets.py from the UNMODIFIED reference `KittiRTM3DDataset._build_target` and
`KittiMonoFlexDataset._build_target` on the constructed label sets of tests/center_targets_cases.py (both detectors, 384x1280 and
375x1242).  The datasets are built by their own constructors over an empty imdb.

Every coordinate derived from the float32 projection (keypoints, MonoFlex's centre) is kept at least 1e-3 heatmap px from an integer, so
an ulp of difference between torch's CPU sin / cos / atan2 and the kernels' cannot change a truncated index: an object that comes closer
is nudged along x and y and projected again (coordinates beyond 4096 px decide no index and are not checked).  The exact_hm_w case is exempt: its projection has no rounded trigonometry.  The generator asserts
that every branch the cases exist for is reached.  Per case: the inputs (mode, image size, P2, objects, classes), whether the reference
raised, and every target array.   python tests/golden/make_golden_center_targets.py"""
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.dirname(HERE), ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import refload  # noqa: E402
import center_targets_cases as cases  # noqa: E402

MARGIN = 1e-3


def datasets():
    refload.load_reference()
    from visualDet3D.data.kitti.dataset.KM3D_dataset import KittiMonoFlexDataset, KittiRTM3DDataset
    tmp = tempfile.mkdtemp()
    os.makedirs(os.path.join(tmp, "training"))
    with open(os.path.join(tmp, "training", "imdb.pkl"), "wb") as f:
        pickle.dump([], f)
    cfg = refload.EasyDict({"path": {"preprocessed_path": tmp}, "obj_types": cases.OBJ_TYPES,
                            "data": {"train_augmentation": [], "test_augmentation": []}})
    return KittiRTM3DDataset(cfg, "training"), KittiMonoFlexDataset(cfg, "training")


def project(ds, rows, P2):
    """The reference's own float32 projection of the objects: (homo_corner / 4 [N, nc, 2], abs_corner z [N, nc])."""
    from visualDet3D.utils.utils import theta2alpha_3d
    if not rows:
        return np.zeros((0, 11, 2), np.float32), np.zeros((0, 11), np.float32)
    b = torch.tensor([[r[0], r[1] - 0.5 * r[4], r[2], r[3], r[4], r[5], theta2alpha_3d(r[6], r[0], r[2], P2)] for r in rows],
                     dtype=torch.float32)
    abs_c, homo, _ = ds.projector.forward(b, torch.tensor(P2, dtype=torch.float32))
    return homo[:, :, 0:2].numpy() / 4, abs_c[:, :, 2].numpy()


def near_int(a):
    """Within MARGIN of an integer; coordinates far outside the map (|v| >= 4096, where a float32 ulp reaches 1e-3) decide nothing."""
    return (np.abs(a - np.round(a)) < MARGIN) & (np.abs(a) < 4096)


def main():
    km3d, monoflex = datasets()
    from visualDet3D.networks.utils.rtm3d_utils import gaussian_radius
    out = {}
    seen = set()
    allc = cases.build_cases()
    out["n_cases"] = np.array(len(allc))
    for ci, (name, mode, H, W, P2, objs) in enumerate(allc):
        ds = monoflex if mode == 1 else km3d
        rows = [list(r) for r, _ in objs]
        cls = [c for _, c in objs]
        if name != "exact_hm_w":
            for _ in range(50):
                ver, _ = project(ds, rows, P2)
                bad = [k for k in range(len(rows)) if near_int(ver[k]).any()]
                if not bad:
                    break
                for k in bad:
                    rows[k][0] += 0.013
                    rows[k][1] += 0.007
            else:
                raise RuntimeError(f"{name}: could not keep the projection off integers")
        labels = [cases.Obj(r, c) for r, c in zip(rows, cls)]
        pre = f"c{ci}/"
        out[pre + "name"] = np.array(name)
        out[pre + "mode"] = np.array(mode)
        out[pre + "hw"] = np.array([H, W])
        out[pre + "P2"] = np.asarray(P2, np.float64)
        out[pre + "objs"] = np.array(rows, np.float64).reshape(-1, 11)
        out[pre + "cls"] = np.array(cls, np.int32)
        try:
            t = ds._build_target(np.zeros((H, W, 3), np.float32), P2.copy(), labels)
        except IndexError:
            assert len(rows) > 32
            out[pre + "raises"] = np.array(1)
            seen.add("over32_raises")
            continue
        out[pre + "raises"] = np.array(0)
        out[pre + "keys"] = np.array(list(t.keys()))
        for k, v in t.items():
            out[pre + "t/" + k] = v
        # which branches this case reaches
        hm_h, hm_w = H // 4, W // 4
        n = len(rows)
        ver, az = project(ds, rows, P2)
        if n == 0:
            seen.add("empty")
        if n == 32:
            seen.add("cap32")
        if H % 4 or W % 4:
            seen.add("size_not_multiple_of_4")
        for k in range(n):
            r = rows[k]
            bb = np.clip(np.array(r[7:11]) / 4, 0, [hm_w, hm_h, hm_w, hm_h])
            valid = bb[3] - bb[1] > 0 and bb[2] - bb[0] > 0
            if not valid:
                seen.add("zero_clipped_bbox")
                continue
            radius = max(0, int(gaussian_radius((np.ceil(bb[3] - bb[1]), np.ceil(bb[2] - bb[0])))))
            if radius == 0 and t["reg_mask"][k]:
                seen.add("radius0")
            seen.add({(1, 0): "rotbin_10", (0, 1): "rotbin_01", (1, 1): "rotbin_11"}[tuple(t["rotbin"][k])])
            K = 10 if mode else 9
            centre = ver[k, 10] if mode else np.array([(bb[0] + bb[2]) / 2, (bb[1] + bb[3]) / 2], np.float32)
            if not t["reg_mask"][k]:
                assert t["location"][k].any()
                seen.add(f"m{mode}_centre_outside")
                if mode and centre[0] >= hm_w:
                    seen.add("monoflex_centre_beyond_hm_w")
                continue
            if mode == 0 and (centre == np.round(centre)).any():
                seen.add("km3d_centre_on_integer")
            if mode and (-1 < centre[0] < 0 or -1 < centre[1] < 0):
                seen.add("monoflex_centre_in_(-1,0)")
            splats = [(int(centre[0]), int(centre[1]))]
            for j in range(K):
                v = ver[k, j]
                if not t["hp_mask"][k * K + j]:
                    seen.add(f"m{mode}_keypoint_outside")
                else:
                    splats.append((int(v[0]), int(v[1])))
                    if ((-1 < v) & (v < 0)).any():
                        seen.add(f"m{mode}_keypoint_in_(-1,0)")
                if mode and v[0] == hm_w:
                    seen.add("monoflex_keypoint_at_hm_w")
                if mode and az[k, j] <= 0:
                    seen.add("monoflex_keypoint_behind_camera")
            for x, y in splats:
                if radius > 0:
                    if x - radius < 0:
                        seen.add(f"m{mode}_clip_left")
                    if x + radius >= hm_w:
                        seen.add(f"m{mode}_clip_right")
                    if y - radius < 0:
                        seen.add(f"m{mode}_clip_top")
                    if y + radius >= hm_h:
                        seen.add(f"m{mode}_clip_bottom")
        cen = [(k, cls[k], t["ind"][k]) for k in range(n) if t["reg_mask"][k]]
        for a in cen:
            for b in cen:
                if a[0] < b[0] and a[1] == b[1] and abs(int(a[2]) - int(b[2])) < 8:
                    seen.add(f"m{mode}_same_class_overlap")
    need = {"empty", "cap32", "over32_raises", "size_not_multiple_of_4", "zero_clipped_bbox", "radius0", "rotbin_10", "rotbin_01",
            "rotbin_11", "km3d_centre_on_integer", "monoflex_centre_in_(-1,0)", "monoflex_centre_beyond_hm_w", "m1_centre_outside",
            "m0_keypoint_in_(-1,0)", "monoflex_keypoint_at_hm_w", "monoflex_keypoint_behind_camera"}
    for m in (0, 1):
        need |= {f"m{m}_keypoint_outside", f"m{m}_same_class_overlap"} | {f"m{m}_clip_{s}" for s in ("left", "right", "top", "bottom")}
    missing = need - seen
    assert not missing, f"branches not reached: {sorted(missing)}"
    np.savez_compressed(os.path.join(HERE, "center_targets.npz"), **out)
    print(f"wrote center_targets.npz: {len(allc)} cases, branches {sorted(seen)}")


if __name__ == "__main__":
    main()
