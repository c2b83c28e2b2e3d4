"""Helpers shared by the tools/bench_*.py scripts: the card a number was measured on, and the timing of one training step."""
import subprocess
import time

import torch


def card():
    """The card's name, power limit and max SM clock (nvidia-smi), which belong beside every number measured on it."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def timed(step, steps, warmup):
    """ms per step() (host clock around `steps` steps ending in a device synchronise, after `warmup`), and from one profiled step: kernel
    launches (memsets included), device-to-host copies and host synchronisations."""
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    launches = sum(("LaunchKernel" in n) or n in ("cudaMemsetAsync",) for n in names)
    d2h = sum(n.startswith("Memcpy DtoH") for n in names)
    syncs = sum(n in ("cudaStreamSynchronize", "cudaDeviceSynchronize") for n in names)
    return dict(ms_per_step=round(ms, 4), launches=launches, d2h_copies=d2h, host_syncs=syncs - 1)    # minus the profiler's own
