"""Hand-written KITTI label / result scenes at the evaluator's decision edges, run through the UNMODIFIED reference evaluator exactly as
make_golden_kitti_eval.py runs its random ones (same stored keys).  python tests/golden/make_golden_kitti_eval_edges.py  ->  kitti_eval_edges.npz

2-D boxes sit on an integer pixel grid, so the float64 bbox overlaps are exact and ties and at-threshold cases are decidable: 14 / 20 is the
double 0.7 and 6 / 12 is 0.5, the minimum overlaps of Car and of Pedestrian.  The lenient table's 0.25 applies to BEV / 3-D only, where the
reference's simulator mixes float64 into the float32 algorithm, so no scene puts a BEV / 3-D overlap at a threshold: object k of an image gets a
3-D box of its own, 6 m from its neighbours, and the `margin` key is kept.  Image "bev" carries rotated pairs at KITTI range (identical at
angle 0, a turned pair, a contained box) and the (-1000, -1, -10) placeholder a 2-D detector writes.  Both cases have fewer than 50 images, so
the reference's overlap computation runs as one part (run_reference's one_part), which it needs below 50 images.
"""
import os

import numpy as np

import make_golden_kitti_eval as G

CAR = (3.9, 1.55, 1.65)                                                    # l, h, w


def box3d(k, gt):
    """The k-th 3-D box of an image: detections on a 6 m x 8 m lattice, ground truth 0.4 m + and 0.05 rad off it."""
    x, z, ry = 6.0 * (k % 10) - 30, 10.0 + 8 * (k // 10), 0.1 * (k % 30)
    return ((x + 0.4 + 0.01 * (k % 7), 1.6, z + 0.3), ry + 0.05) if gt else ((x, 1.6, z), ry)


class Image:
    def __init__(self):
        self.gts, self.dts = [], []

    def gt(self, name, x1, y1, w, h, trunc=0.0, occ=0, dims=CAR, loc=None, ry=None):
        k = len(self.gts)
        l, r = box3d(k, True)
        if name == "DontCare":
            o = dict(name=name, trunc=-1.0, occ=-1, alpha=-10.0, bbox=(x1, y1, x1 + w, y1 + h), dims=(-1.0, -1.0, -1.0),
                     loc=(-1000.0, -1000.0, -1000.0), ry=-10.0)
        else:
            o = dict(name=name, trunc=trunc, occ=occ, alpha=0.1 * (k % 30), bbox=(x1, y1, x1 + w, y1 + h), dims=dims, loc=loc or l,
                     ry=r if ry is None else ry)
        self.gts.append(G.label_line(o) + "\n")
        return self

    def dt(self, name, x1, y1, w, h, score, dims=CAR, loc=None, ry=None):
        k = len(self.dts)
        l, r = box3d(k, False)
        self.dts.append(G.result_line(name, 0.1 * (k % 30) + 0.05, (x1, y1, x1 + w, y1 + h), dims, loc or l, r if ry is None else ry, score))
        return self


def scenes():
    im = {}
    s = im["thr_car"] = Image()                                             # Car, 17 px wide: shifts 3 / 2 / 4 px give 14/20, 15/19, 13/21
    for k, shift in enumerate((3, 2, 4)):
        s.gt("Car", 100 + 200 * k, 150, 17, 50).dt("Car", 100 + 200 * k + shift, 150, 17, 50, 0.9 - 0.1 * k)
    s = im["thr_ped"] = Image()                                             # Pedestrian, 9 px wide: 6/12, 7/11, 5/13; Cyclist has no ground truth anywhere
    for k, shift in enumerate((3, 2, 4)):
        s.gt("Pedestrian", 100 + 100 * k, 150, 9, 60).dt("Pedestrian", 100 + 100 * k + shift, 150, 9, 60, 0.85 - 0.1 * k)
        s.dt("Cyclist", 600 + 100 * k, 150, 30, 60, 0.5)
    s = im["ties"] = Image()
    s.gt("Car", 100, 150, 17, 50).dt("Car", 102, 150, 17, 50, 0.6).dt("Car", 98, 150, 17, 50, 0.8)           # equal overlaps, different scores
    s.gt("Car", 300, 150, 17, 50).dt("Car", 302, 150, 17, 50, 0.5).dt("Car", 298, 150, 17, 50, 0.5)          # equal overlaps, equal scores
    s.gt("Car", 500, 150, 17, 50).gt("Car", 504, 150, 17, 50).dt("Car", 502, 150, 17, 50, 0.7)               # two ground truths, one detection
    for n in ("same_score_a", "same_score_b"):                              # equal scores across images
        im[n] = Image().gt("Car", 100, 150, 60, 50).dt("Car", 101, 150, 60, 50, 0.75).gt("Car", 300, 150, 60, 50).dt("Car", 300, 151, 60, 50, 0.65)
    s = im["heights"] = Image()                                             # minimum heights 40 / 25 / 25: `<=` for ground truth, `<` for detections
    for k, (hg, hd) in enumerate(((40, 40), (41, 41), (25, 25), (26, 26), (42, 40), (42, 39), (26, 25), (26, 24))):
        s.gt("Car", 50 + 140 * k, 100, 80, hg).dt("Car", 50 + 140 * k, 100, 80, hd, 0.95 - 0.05 * k)
    s = im["occ_trunc"] = Image()                                           # maximum occlusion 0 / 1 / 2, truncation 0.15 / 0.30 / 0.50 (`>` ignores)
    for k, (occ, tr) in enumerate(((0, 0.0), (1, 0.0), (2, 0.0), (3, 0.0), (0, 0.15), (0, 0.16), (0, 0.30), (0, 0.31), (0, 0.50), (0, 0.51))):
        s.gt("Car", 20 + 120 * k, 100, 80, 60, trunc=tr, occ=occ).dt("Car", 20 + 120 * k, 101, 80, 60, 0.9 - 0.03 * k)
    s = im["dontcare"] = Image()
    s.gt("DontCare", 100, 100, 100, 50).gt("Car", 400, 100, 80, 60).gt("Van", 600, 100, 80, 60).gt("DontCare", 690, 100, 100, 60)
    s.dt("Car", 120, 102, 40, 45, 0.9)                                      # inside the region
    s.dt("Car", 186, 102, 20, 45, 0.8).dt("Car", 185, 104, 20, 45, 0.7)     # 14 / 20 of the detection inside (not above 0.7), then 15 / 20
    s.dt("Car", 400, 101, 80, 60, 0.85).dt("Car", 601, 100, 80, 60, 0.6)    # the Car, and one on the Van
    s.dt("Car", 640, 100, 80, 60, 0.55)                                     # half on the Van (below 0.7), 30 / 80 in the second region
    im["gt_only"] = Image().gt("Car", 100, 100, 80, 60).gt("Pedestrian", 300, 100, 30, 70)
    im["dt_only"] = Image().dt("Car", 100, 100, 80, 60, 0.4).dt("Pedestrian", 300, 100, 30, 70, 0.3)
    im["empty"] = Image()
    s = im["seventy"] = Image()                                             # 70 detections = three 32-bit flag words; 45 matches in words 0, 1, 2
    for j in range(70):
        s.dt("Car", 20 + 110 * (j % 10), 10 + 50 * (j // 10), 60, 45, round(0.99 - 0.01 * j, 2))
    for j in list(range(0, 15)) + list(range(32, 47)) + list(range(55, 70)):
        s.gt("Car", 21 + 110 * (j % 10), 10 + 50 * (j // 10), 60, 45)
    s = im["bev"] = Image()
    s.gt("Car", 100, 100, 80, 60, dims=(4.0, 1.5, 2.0), loc=(40.0, 1.6, 78.0), ry=0.0).dt("Car", 100, 100, 80, 60, 0.9, dims=(4.0, 1.5, 2.0), loc=(40.0, 1.6, 78.0), ry=0.0)
    s.gt("Car", 300, 100, 80, 60, dims=(4.0, 1.5, 2.0), loc=(-25.0, 1.6, 45.0), ry=0.4).dt("Car", 300, 100, 80, 60, 0.8, dims=(4.0, 1.5, 2.0), loc=(-25.0, 1.6, 45.0), ry=0.9)
    s.gt("Car", 500, 100, 80, 60, dims=(6.0, 1.5, 5.0), loc=(0.0, 1.6, 30.0), ry=0.4).dt("Car", 500, 100, 80, 60, 0.7, dims=(2.0, 1.5, 1.0), loc=(0.5, 1.6, 30.5), ry=1.7)
    s.gt("DontCare", 700, 100, 50, 50).dt("Car", 900, 100, 80, 60, 0.6, dims=(-1, -1, -1), loc=(-1000, -1000, -1000), ry=-10)
    return im


def main():
    G.refload.load_reference()
    import visualDet3D.evaluator.kitti.eval as E
    import visualDet3D.evaluator.kitti.evaluate as KE
    import visualDet3D.evaluator.kitti.kitti_common as KC
    im = scenes()
    names = list(im)
    out = {"edges/scenes": np.array(names)}
    for case, pick in (("edges", names), ("single", ["thr_car"])):
        ids = np.arange(len(pick)) * 7 + 3
        labels, results = ["".join(im[n].gts) for n in pick], ["".join(im[n].dts) for n in pick]
        texts, captured, ious, gt_annos, dt_annos = G.run_reference(E, KE, KC, ids, labels, results, (0, 1, 2), True)
        ng, nd = G.store_case(out, case, ids, labels, results, (0, 1, 2), texts, captured, ious, gt_annos, dt_annos)
        margin = float(out[case + "/margin"])
        assert margin > G.MARGIN, f"{case}: a BEV / 3-D overlap within {margin:.3g} of a threshold or of another one"
        print(f"{case}: {len(ids)} images, {ng.sum()} gt, {nd.sum()} dt, margin {margin:.3g}")
        print(texts[0])
    np.savez_compressed(os.path.join(G.HERE, "kitti_eval_edges.npz"), **out)


if __name__ == "__main__":
    main()
