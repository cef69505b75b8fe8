"""Scaffolding shared by the benchmark tools: the card's identity, the device check, per-arm statistics, the alternating timer and the A/B
against another build of the library.  Importing it puts the repository root and tests/ (gpu_harness, helpers) on sys.path."""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def card():
    """the card's name, power limit and maximum SM clock (read-only nvidia-smi query)"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def device_lib(tool):
    """capi.lib(), or exit where no CUDA device is visible"""
    import dmvio_b200.capi as capi
    L = capi.lib()
    if L.dmv_device_count() < 1:
        raise SystemExit(f"{tool} needs a CUDA device")
    return L


def stats(ts):
    """median / p10 / p90 in ms of wall times in s; the caller adds its rate fields"""
    ms = 1e3 * np.asarray(ts)
    return dict(median_ms=float(np.median(ms)), p10_ms=float(np.percentile(ms, 10)), p90_ms=float(np.percentile(ms, 90)))


def alternate(arms, warmup, reps, what, libs, resets=None):
    """times arms (name -> call returning a dmv_status) in warmup + reps repetitions; each repetition calls every arm once, starting one arm
    later than the one before, and the first `warmup` are not kept.  resets[name] runs before its arm, outside the timing.  A non-zero
    status exits with the message of libs[name].  Returns name -> wall times in s."""
    names = list(arms)
    t = {k: [] for k in names}
    for rep in range(warmup + reps):
        for j in range(len(names)):
            k = names[(rep + j) % len(names)]
            if resets:
                resets[k]()
            t0 = time.perf_counter()
            rc = arms[k]()
            dt = time.perf_counter() - t0
            if rc != 0:
                raise SystemExit(f"{k} {what}: dmvio_b200 error {rc}: {libs[k].dmv_last_error().decode()}")
            if rep >= warmup:
                t[k].append(dt)
    return t


def this_and_parent(path):
    """{"this": this build's library, "parent": the build at `path`, e.g. the parent commit's}, bound alike, for an A/B in one process"""
    import dmvio_b200.capi as capi
    return {"this": capi.lib(), "parent": capi.load(path)}
