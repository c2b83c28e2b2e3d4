"""Checks shared by the GPU training-loss tests (tests/test_*loss_gpu.py); not collected by pytest."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def graph_replay_matches_eager(step):
    """Run step() (a forward + backward returning the tensors to compare) once eagerly on a side stream, capture it in a CUDA graph, and
    assert two replays reproduce the eager tensors bit for bit."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = [t.clone() for t in step()]
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step()
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(outs, eager):
            assert torch.equal(x, y)


def run_seam_worker(script, *args, timeout=900):
    """Run tests/workers/<script> with args and return the JSON of its last `SEAM_JSON ` line; skip without the reference package."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import refload
    if not refload.available():
        pytest.skip("no reference package (neither the reference tree nor oracle/_ref/visualDet3D)")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "workers", script), *args], capture_output=True, text=True,
                       timeout=timeout)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("SEAM_JSON ")]
    assert r.returncode == 0 and lines, f"worker failed (rc {r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    out = json.loads(lines[-1][len("SEAM_JSON "):])
    print(out)
    return out
