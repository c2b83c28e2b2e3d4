"""-m gpu: Stereo3D's cost-volume kernels on the constructed cases of tests/cost_volume_cases.py, against its float64 restatements.

Paths (the kernel the launch rules of engine.psm_cosine_stereo and vd3d_psm_cosine_nhwc pick for each case):
  * tc       psm_cosine_tc_kernel (csrc/psm_tc.cu) through engine.psm_cosine_stereo, with the fp16 planes refreshed by the call and
             supplied fresh (the fp32 tensor then holds NaN: the kernel must read the planes only);
  * v4       psm_cosine_nhwc_v4_kernel, C = 64 and C = 128, several 64-pixel tiles per persistent CTA;
  * v3       psm_cosine_nhwc_v3_kernel, reached with the default variant by channel-sliced inputs;
  * v2, v3   on dense inputs under VD3D_PSM_VARIANT = 2 / 3, in a worker process (tests/workers/psm_variant.py): the variant is read once
             per process;
  * generic  psm_cosine_nhwc_generic_kernel: D != 24, C = 32, an output pitch / offset that is not a multiple of 4;
  * nchw     psm_cosine_nchw_kernel;
  * concat   concat_conv3d_1_kernel + conv3d_2_kernel.
Every case runs twice: integer tag operands, compared bit for bit, and random fp32 operands, held to the per-element bounds derived in
cost_volume_cases.py (the ratio |error| / bound must stay <= 1).  Every run also checks the w < d triangle is exactly 0, the output channels
around the written slice keep their sentinel, and a second launch into the same buffer reproduces the first bit for bit.  Each case prints
its path, tiles per CTA, the largest random-case error and its ratio to the bound.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

import cost_volume_cases as cv
from visualdet3d_b200 import engine as E
from visualdet3d_b200._lib import call

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUM_SMS = 132                  # H100 SXM: the persistent grids are min(tiles, 132) (tc, v4 at C = 128) or min(tiles, 264) (v4 at C = 64)
SENT = -7.25


def tiles_per_cta(path, case):
    B, H, W, C = case["B"], case["H"], case["W"], case["C"]
    if path == "tc":
        n = math.ceil(B * H * W / cv.TC_TILE)
        return math.ceil(n / min(n, NUM_SMS))
    if path == "v4":
        n = B * H * math.ceil(W / 64)
        return math.ceil(n / min(n, NUM_SMS * (2 if C == 64 else 1)))
    return 1


def _valid(B, H, W, D):
    w = torch.arange(W, device="cuda").reshape(1, 1, W, 1)
    return (w >= torch.arange(D, device="cuda").reshape(1, 1, 1, D)).expand(B, H, W, D)


def check_run(launch, out, ret=None):
    """Launch and check it returned `ret`; launch again into the same buffer (same bits); check the sentinels around the output slice.
    Returns the slice."""
    r = launch()
    assert ret is None or r == ret, (r, ret)
    first = out.t.clone()
    launch()
    torch.cuda.synchronize()
    assert torch.equal(out.t, first), "second launch into the same buffer differs"
    assert bool((out.t[..., :out.co] == SENT).all()) and bool((out.t[..., out.co + out.C:] == SENT).all()), "sentinel channels overwritten"
    return out.t[..., out.co:out.co + out.C]


def compare_psm(got, L, R, case, tag, bound_fn, path):
    """Exact (tag) or bounded (random) comparison of a [B, H, W, D] result; returns (max |err|, max |err| / bound)."""
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    want, S = cv.psm_cosine64(L.cuda(), R.cuda(), D)
    assert bool((got[~_valid(B, H, W, D)] == 0).all()), "w < d triangle not exactly 0"
    assert bool(torch.isfinite(got).all())
    if tag:
        exp = cv.device_scale(want, C, divide=path in ("generic", "nchw"))
        bad = int((got != exp).sum())
        assert bad == 0, f"{bad} of {got.numel()} tag elements differ, first at {(got != exp).nonzero()[0].tolist()}"
        return 0.0, 0.0
    err = (got.double() - want).abs()
    ratio = ratio_of(err, bound_fn(S))
    assert ratio <= 1.0, ratio
    return float(err.max()), ratio


def ratio_of(err, bound):
    """max err / bound, where a zero bound (a restated element with no terms) admits only a zero error."""
    return float((err / bound.clamp_min(1e-300)).max())


def report(path, case, err, ratio):
    print(f"  {path:8s} {case['id']:20s} tiles/CTA {tiles_per_cta(path, case)}  max|err| {err:.3e}  max|err|/bound {ratio:.3e}")


def planes(shape, fill):
    return torch.full((2, *shape), fill, device="cuda", dtype=torch.float16)


# ---- tensor-core PSMCosine --------------------------------------------------------------------------------------------------------------
def run_tc(case, L, R, planes_fresh):
    B, H, W, C, D, cs, co = (case[k] for k in ("B", "H", "W", "C", "D", "cs", "co"))
    lr = torch.cat([L, R]).cuda()
    t = torch.full((2 * B, H, W, cs), 3.0, device="cuda")
    pl = planes((2 * B, H, W, cs), 5.0)
    if planes_fresh:
        hi, lo = E.fp16_split(lr)
        pl[0, ..., co:co + C], pl[1, ..., co:co + C] = hi, lo
        t[..., co:co + C] = float("nan")
    else:
        t[..., co:co + C] = lr
    f = E.Act(t, co, C, pl)
    out = E.Act(torch.full((B, H, W, case["out_cs"]), SENT, device="cuda"), case["out_co"], D)
    return check_run(lambda: E.psm_cosine_stereo(f, B, D, out, planes_fresh=planes_fresh), out, ret=not planes_fresh)


@pytest.mark.parametrize("planes_fresh", [False, True])
@pytest.mark.parametrize("case", cv.TC_CASES, ids=[c["id"] for c in cv.TC_CASES])
def test_psm_tensor_core(case, planes_fresh):
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    L, R = cv.tag_features(B, H, W, C, cv.case_seed(case))
    compare_psm(run_tc(case, L, R, planes_fresh), L, R, case, True, None, "tc")
    L, R = cv.random_features(B, H, W, C, cv.case_seed(case))
    Lc, Rc = L.cuda(), R.cuda()
    err, ratio = compare_psm(run_tc(case, L, R, planes_fresh), L, R, case, False, lambda S: cv.tc_bound(C, S, Lc, Rc), "tc")
    report("tc", case, err, ratio)


# ---- SIMT PSMCosine ---------------------------------------------------------------------------------------------------------------------
def run_simt(case, L, R):
    B, H, W, C, D, cs, co = (case[k] for k in ("B", "H", "W", "C", "D", "cs", "co"))
    acts = []
    for x in (L, R):
        t = torch.full((B, H, W, cs), 3.0, device="cuda")
        t[..., co:co + C] = x.cuda()
        acts.append(E.Act(t, co, C))
    out = E.Act(torch.full((B, H, W, case["out_cs"]), SENT, device="cuda"), case["out_co"], D)
    return check_run(lambda: E.psm_cosine(acts[0], acts[1], D, out), out)


def check_simt_case(case, path):
    """Tag and random runs of one SIMT case on `path`; returns (max |err|, max ratio) of the random run (also used by the variant worker)."""
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    L, R = cv.tag_features(B, H, W, C, cv.case_seed(case))
    compare_psm(run_simt(case, L, R), L, R, case, True, None, path)
    L, R = cv.random_features(B, H, W, C, cv.case_seed(case))
    err, ratio = compare_psm(run_simt(case, L, R), L, R, case, False, lambda S: cv.simt_bound(C, S), path)
    report(path, case, err, ratio)
    return err, ratio


@pytest.mark.parametrize("case", cv.SIMT_CASES, ids=[c["id"] for c in cv.SIMT_CASES])
def test_psm_simt(case):
    check_simt_case(case, case["path"])


@pytest.mark.parametrize("variant", [2, 3])
def test_psm_simt_env_variants(variant):
    env = dict(os.environ, VD3D_PSM_VARIANT=str(variant))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "workers", "psm_variant.py")], capture_output=True, text=True,
                       timeout=600, env=env)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("PSM_JSON ")]
    assert r.returncode == 0 and lines, f"worker failed (rc {r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    print(r.stdout)
    res = json.loads(lines[-1][len("PSM_JSON "):])
    assert res["path"] == f"v{variant}" and sorted(res["cases"]) == sorted(c["id"] for c in cv.VARIANT_CASES)
    assert all(rec["ratio"] <= 1.0 for rec in res["cases"].values())


@pytest.mark.parametrize("case", cv.NCHW_CASES, ids=[c["id"] for c in cv.NCHW_CASES])
def test_psm_nchw(case):
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    n = B * D * H * W
    for tag in (True, False):
        L, R = (cv.tag_features if tag else cv.random_features)(B, H, W, C, cv.case_seed(case))
        Ln, Rn = (x.permute(0, 3, 1, 2).contiguous().cuda() for x in (L, R))
        buf = torch.full((n + 64,), SENT, device="cuda")
        out = E.Act(buf.reshape(1, 1, 1, -1), 0, n)          # the dense [B, D, H, W] result, sentinels after it
        launch = lambda: call("vd3d_psm_cosine_nchw", Ln.data_ptr(), Rn.data_ptr(), B, C, H, W, D, buf.data_ptr(), E._stream())  # noqa: E731
        got = check_run(launch, out).reshape(B, D, H, W).permute(0, 2, 3, 1)
        err, ratio = compare_psm(got, L, R, case, tag, lambda S: cv.simt_bound(C, S), "nchw")
    report("nchw", case, err, ratio)


# ---- concat volume + Conv3d pair ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", cv.CONCAT_CASES, ids=[c["id"] for c in cv.CONCAT_CASES])
def test_concat_volume_conv3d(case):
    B, H, W, Fc, D = case["B"], case["H"], case["W"], case["F"], case["D"]
    for tag in (True, False):
        ops = (cv.tag_conv_operands if tag else cv.random_conv_operands)(B, H, W, Fc, cv.case_seed(case, 1 if tag else 0))
        lf, rf, w1, b1, w2, b2 = ops
        lr = torch.cat([lf, rf]).cuda()                      # one [2B] tensor, left then right, as the down-sample conv writes it
        dev = [cv.pack_conv3d(w1).cuda(), b1.cuda(), cv.pack_conv3d(w2).cuda(), b2.cuda()]
        mid = torch.full((B, D, H, W, Fc), SENT, device="cuda")
        out = E.Act(torch.full((B, H, W, case["out_cs"]), SENT, device="cuda"), case["out_co"], Fc * D)
        launch = lambda: call("vd3d_concat_volume_conv3d", lr[:B].data_ptr(), lr[B:].data_ptr(), B, H, W, Fc, D,  # noqa: E731
                              *(t.data_ptr() for t in dev), mid.data_ptr(), out.ptr, out.cs, out.co, E._stream())
        got = check_run(launch, out)
        r = cv.concat_conv3d64(*(t.cuda() for t in ops), D)
        if tag:
            bad = int((got.double() != r["out"]).sum())
            assert bad == 0, f"{bad} of {got.numel()} tag elements differ"
            assert torch.equal(mid.double(), r["mid"].permute(0, 2, 3, 4, 1)), "Conv3d #1 output differs"
        else:
            err = (got.double() - r["out"]).abs()
            ratio = ratio_of(err, r["bound"])
            assert ratio <= 1.0, ratio
            report("concat", dict(case, C=2 * Fc), float(err.max()), ratio)
