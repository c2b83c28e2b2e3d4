"""SHA-256 digests of the test-time input pipeline's output (`preprocess.preprocess_host`) -> tests/golden/preprocess_digests.npz, on:
  * the 10 frames / 5 geometries of tests/golden/preprocess.npz (`make_golden_preprocess.frame`, the RGB_MEAN / RGB_STD Normalize);
  * every plain-resize case of tests/augment_cases.py (no photometric program; a mirrored case's frame is taken unmirrored, since the
    test-time pipeline has no mirror);
  * seeded 375 x 1242 frames at the two bench.py geometries: crop 2 -> 384 x 1280 and crop 96 -> 288 x 1280.
The fixture tests hold the pipeline to 2e-5 of the reference; the digests pin every output bit, so a change to how the resize is computed
must reproduce them exactly.  The host entry runs on the CPU, no GPU is needed:

    python tests/golden/make_golden_preprocess_digests.py

`tests/test_preprocess_digests_cpu.py` and `tests/test_preprocess_digests_gpu.py` import `cases`, `OUT` and `digest`."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "preprocess_digests.npz")
for _p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

BENCH_GEOMETRIES = ((2, (384, 1280)), (96, (288, 1280)))        # bench.py: 375 x 1242 frames, crop_top = 375 - round(1242 * H / W)


def cases():
    """-> [{id, frame, crop_top, size, mean, std}], the inputs of every digest."""
    import augment_cases as ac
    from make_golden_preprocess import frame
    from visualdet3d_b200.preprocess import RGB_MEAN, RGB_STD
    out = []
    fx = np.load(os.path.join(ROOT, "tests", "golden", "preprocess.npz"))
    for ci in range(len([k for k in fx.files if k.endswith("_meta")])):
        seed, H, W, crop, Ho, Wo = [int(v) for v in fx[f"c{ci}_meta"]]
        for side, sd in (("l", seed), ("r", seed + 100)):
            out.append(dict(id=f"fixture/c{ci}_{side}", frame=frame(sd, H, W), crop_top=crop, size=(Ho, Wo), mean=RGB_MEAN, std=RGB_STD))
    for c in ac.CASES:
        if c["geom"] == ac.GEOM_RESIZE and len(c["ops"]) == 0:
            out.append(dict(id=f"resize/{c['id']}", frame=c["frame"], crop_top=c["crop_top"], size=(c["Ho"], c["Wo"]), mean=ac.MEAN, std=ac.STD))
    for crop, size in BENCH_GEOMETRIES:
        for seed in (0, 1):
            img = np.random.RandomState(100 + seed).randint(0, 256, (375, 1242, 3)).astype(np.uint8)
            out.append(dict(id=f"bench/crop{crop}_{size[0]}x{size[1]}_s{seed}", frame=img, crop_top=crop, size=size, mean=RGB_MEAN, std=RGB_STD))
    return out


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    from visualdet3d_b200 import preprocess as pp
    fx = {}
    for c in cases():
        got = pp.preprocess_host(c["frame"], c["crop_top"], c["size"], c["mean"], c["std"])
        fx[c["id"]] = np.array(digest(got))
        print(c["id"], got.shape, fx[c["id"]], flush=True)
    np.savez(OUT, **fx)
    print("wrote", OUT, len(fx), "digests")


if __name__ == "__main__":
    main()
