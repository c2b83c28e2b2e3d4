"""Worker of tests/test_center_targets_gpu.py::test_plugin_matches_the_reference_training_input (own process, GPU box).

Writes the two-frame KITTI tree of tests/workers/train_augment_plugin.py under argv[1] and runs, from the same numpy seed, the reference's
KittiRTM3DDataset (KM3D_example's list) and KittiMonoFlexDataset (MonoFlex_example's list) + collate_fn + train_rtm3d into a recording
stub module: as shipped, after `plugin.install_train_targets_into_reference()`, and after `install_train_augmentation_into_reference()` as
well.  Prints one JSON line: per dataset and arm, whether the module got the shipped run's keys, dtypes and shapes, bit-equal integer /
mask / heatmap targets, float targets within the host-form rules (tests/test_center_targets_cpu.py), the targets on the GPU, equal P2, the
largest image difference, and whether the numpy RNG ends at the same position."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "workers")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import refload  # noqa: E402
import train_augment_cases as cases  # noqa: E402
from train_augment_plugin import SIZES, write_tree  # noqa: E402

PROJECTED = ("hps", "hp_offset", "reg")


class Recorder(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1, device="cuda"))
        self.seen = None

    def forward(self, inputs):
        image, gts, meta = inputs
        self.seen = {"image": image.detach().float().cpu(), "on_gpu": all(v.is_cuda for v in gts.values()),
                     "gts": {k: v.cpu() for k, v in gts.items()}, "P2": meta["P2"].cpu()}
        s = self.p.sum()
        return s + 1.0, {}


def run(cfg, ds_cls, seed):
    from visualDet3D.networks.utils import registry as ref
    ds = ds_cls(cfg, "training")
    np.random.seed(seed)
    data = ds_cls.collate_fn([ds[i] for i in range(len(SIZES))])
    module = Recorder()
    ref.PIPELINE_DICT["train_rtm3d"](data, module, torch.optim.SGD(module.parameters(), lr=0.1), cfg=cfg, epoch_num=0)
    torch.cuda.synchronize()
    return module.seen, np.random.rand()


def compare(seen, nxt, ref_seen, ref_next, hm_w):
    g, r = seen["gts"], ref_seen["gts"]
    keys = list(g) == list(r)
    ds = all(g[k].dtype == r[k].dtype and g[k].shape == r[k].shape for k in r)
    exact = all(torch.equal(g[k], r[k]) for k in r if k in ("hm", "hm_hp") or r[k].dtype != torch.float32)
    close = True
    for k in r:
        if r[k].dtype == torch.float32 and k not in ("hm", "hm_hp"):
            w = r[k].numpy()
            tol = np.maximum(1e-5, 2 * np.spacing(np.abs(w) + np.float32(hm_w))) if k in PROJECTED else 1e-5
            close &= bool((np.abs(g[k].numpy().astype(np.float64) - w) <= tol).all())
    return {"keys_equal": keys, "dtypes_shapes_equal": ds, "exact_equal": exact, "float_close": close, "targets_on_gpu": seen["on_gpu"],
            "P2_equal": torch.equal(seen["P2"], ref_seen["P2"]), "image_max_diff": float((seen["image"] - ref_seen["image"]).abs().max()),
            "rng_equal": nxt == ref_next, "n_keys": len(g)}


def main():
    from visualdet3d_b200 import plugin
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_train_augment import edict
    from visualDet3D.data.kitti.dataset.KM3D_dataset import KittiMonoFlexDataset, KittiRTM3DDataset
    pre = write_tree(sys.argv[1])
    arms = {"km3d": KittiRTM3DDataset, "monoflex": KittiMonoFlexDataset}

    def cfg(name):
        return edict({"path": {"preprocessed_path": pre}, "obj_types": ["Car"],
                      "data": {"augmentation": {}, "train_augmentation": cases.LISTS[name][0], "use_right_image": False},
                      "optimizer": {"clipped_gradient_norm": 1.0}})

    seed = 0
    shipped = {name: run(cfg(name), cls, seed) for name, cls in arms.items()}
    out = {}
    plugin.install_train_targets_into_reference()
    plugin.install_train_targets_into_reference()         # installing twice wraps once
    for name, cls in arms.items():
        out[f"{name}_targets"] = compare(*run(cfg(name), cls, seed), *shipped[name], 1280 // 4)
    plugin.install_train_augmentation_into_reference()
    for name, cls in arms.items():
        out[f"{name}_both"] = compare(*run(cfg(name), cls, seed), *shipped[name], 1280 // 4)
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
