"""ORACLE infrastructure (not product code): copies the reference's det_precompute scripts verbatim into oracle/_ref/scripts (git-ignored,
next to the package copy oracle/build_ref.py makes), so that tools/bench_det_precompute.py and tests/test_det_precompute_gpu.py can run
the unmodified reference script on the GPU box, where the reference tree itself is absent.  Nothing in the product package reads them.

    build()       in the build container (needs the reference tree); a no-op elsewhere
"""
from __future__ import annotations

import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref", "scripts")
REF = os.environ.get("VISUALDET3D_REF", "/root/reference")
SCRIPTS = ("imdb_precompute_3d.py", "imdb_precompute_test.py", "_path_init.py")


def build() -> None:
    src = os.path.join(REF, "scripts")
    if not all(os.path.isfile(os.path.join(src, f)) for f in SCRIPTS):
        return
    os.makedirs(OUT, exist_ok=True)
    for f in SCRIPTS:
        shutil.copyfile(os.path.join(src, f), os.path.join(OUT, f))


if __name__ == "__main__":
    build()
    print(OUT, sorted(os.listdir(OUT)) if os.path.isdir(OUT) else "absent")
