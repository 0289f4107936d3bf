"""The one timing layer of the measurement scripts under tools/: every number they print is taken here, the same way,
with the card's name and power limit beside it.

    require_cuda(what)                        exit with one line when there is no CUDA device (no CPU fallback)
    card()                                    {"name", "power_limit", "max_sm_clock"} of device 0, read once
    cuda_time(fn, reps, warmup=3, batch=1)    CUDA events: each sample is one event pair around `batch` back-to-back
                                              calls, divided by `batch`
    host_time(fn, reps, warmup)               host clock around each call, with a device synchronise before and after
    kernel_times(fn, steps=1, match=None)     device µs per kernel name from one torch.profiler pass
    emit(record, out=None)                    one JSON line with the card merged in, optionally also written to `out`

The timers return {"median_ms", "min_ms", "max_ms", "samples_ms"}.  kernel_times traces, so it never runs inside a
timed window; call it after the timers.
"""
import functools
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch


def require_cuda(what):
    if not torch.cuda.is_available():
        sys.exit("%s: needs a CUDA device" % what)


@functools.lru_cache(maxsize=None)
def card():
    """read-only: one nvidia-smi query, which changes no setting"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
        power_limit, max_sm_clock = (s.strip() for s in q.split(","))
    except Exception as e:  # noqa: BLE001
        power_limit = max_sm_clock = "unknown (%s)" % e
    return {"name": torch.cuda.get_device_name(0), "power_limit": power_limit, "max_sm_clock": max_sm_clock}


def _summary(samples):
    return {"median_ms": float(np.median(samples)), "min_ms": float(np.min(samples)), "max_ms": float(np.max(samples)),
            "samples_ms": [float(s) for s in samples]}


def cuda_time(fn, reps, warmup=3, batch=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    samples = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(batch):
            fn()
        e1.record()
        e1.synchronize()
        samples.append(e0.elapsed_time(e1) / batch)
    return _summary(samples)


def host_time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    samples = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        samples.append(1e3 * (time.perf_counter() - t))
    return _summary(samples)


class KernelTimes(dict):
    """{kernel name: device µs per step}, with `launches` {kernel name: launches per step} and `host_syncs`, the names
    of the host synchronisation calls made in the pass (including the pass's own closing synchronise)"""


def kernel_times(fn, steps=1, match=None):
    """one torch.profiler pass (CPU and CUDA activities) over `steps` calls of fn and a synchronise; copies and memsets
    count as kernels.  match: keep only names containing one of these substrings"""
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = KernelTimes()
    out.launches, out.host_syncs = {}, []
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CPU:
            if "Synchronize" in ev.name:
                out.host_syncs.append(ev.name)
        elif match is None or any(m in ev.name for m in match):
            out[ev.name] = out.get(ev.name, 0.0) + ev.device_time_total / steps
            out.launches[ev.name] = out.launches.get(ev.name, 0) + 1 / steps
    return out


def emit(record, out=None):
    record = dict(record, card=card())
    print(json.dumps(record), flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump(record, f, indent=1)
    return record
