"""Worker of tests/test_cost_volume_cases_gpu.py::test_psm_simt_env_variants (own process, GPU box).

Runs the dense PSMCosine cases (cost_volume_cases.VARIANT_CASES) under the VD3D_PSM_VARIANT its parent set (2 or 3): the launch rules read
the variant once per process, so a test cannot switch it in place.  The checks are the parent module's (`check_simt_case`: the kernel
name, tag cases bit-exact, random cases within the derived bound, triangle, sentinels, a repeated launch); an assertion fails the process.
Prints one PSM_JSON line with the path and each case's largest random-case error and ratio to the bound."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import cost_volume_cases as cv  # noqa: E402
from test_cost_volume_cases_gpu import check_simt_case  # noqa: E402


def main():
    path = "v" + os.environ["VD3D_PSM_VARIANT"]
    assert path in ("v2", "v3"), path
    cases = {}
    for case in cv.VARIANT_CASES:
        err, ratio = check_simt_case(case, path)
        cases[case["id"]] = dict(err=err, ratio=ratio)
    print("PSM_JSON " + json.dumps(dict(path=path, cases=cases)))


if __name__ == "__main__":
    main()
