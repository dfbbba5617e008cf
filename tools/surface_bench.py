#!/usr/bin/env python
"""surface_bench.py — time of the validation surface distances (calculate_distance, metric/utils.py:8-28) on the GPU
against the unmodified reference function on the host CPU, on seeded organ-like label maps of two validation shapes:

  kits  128x256x256, 3 classes  (spacing 2.5, 0.78, 0.78)
  amos   96x256x256, 16 classes (spacing 2.0, 0.7, 0.7)

  python tools/surface_bench.py [--reps 10] [--ref-reps 1] [--cases kits amos] [--out FILE]

GPU: b200seg.calculate_distance on int64 CUDA label maps, two warm-up calls, then --reps calls each ended by a device
synchronise (the call itself returns host numpy arrays, so it always synchronises); median and min are printed.
CPU: metric.utils.calculate_distance imported from oracle/_ref (installed there by the build through
oracle/install_ref_metric.py from the reference checkout), on the same maps copied to the host; "not measured" when it cannot be imported.  numpy >= 2 removed
np.Inf, which the reference uses for empty masks, so the script sets np.Inf = np.inf before importing it.
The GPU name, power limit, CPU model and core count are printed with the numbers, and the two outputs are compared
(nan / inf in the same places, finite values within 1e-9 relative)."""
import argparse
import json
import os
import platform
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import b200seg                                  # noqa: E402
from oracle.surface import synthetic_pair       # noqa: E402

CASES = {"kits": dict(shape=(128, 256, 256), C=3, spacing=(2.5, 0.78, 0.78), seed=1),
         "amos": dict(shape=(96, 256, 256), C=16, spacing=(2.0, 0.7, 0.7), seed=2)}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def cpu_info():
    model = platform.processor() or "unknown"
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                model = line.split(":", 1)[1].strip()
                break
    except OSError:
        pass
    return "%s, %d logical cores" % (model, os.cpu_count() or 0)


def reference_fn():
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.exists(os.path.join(ref, "metric", "utils.py")):
        return None, "oracle/_ref/metric/utils.py missing"
    np.Inf = np.inf
    sys.path.insert(0, ref)
    try:
        import metric.utils as mu
    except Exception as e:          # scipy or another dependency missing on this host
        return None, "%s: %s" % (type(e).__name__, e)
    return mu.calculate_distance, None


def same(a, b):
    return (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isinf(a), np.isinf(b))
            and np.allclose(a[np.isfinite(a)], b[np.isfinite(b)], rtol=1e-9, atol=0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ref-reps", type=int, default=1)
    ap.add_argument("--cases", nargs="+", default=list(CASES))
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "surface_bench needs a CUDA device"
    print("GPU: %s" % gpu_info())
    print("CPU: %s" % cpu_info())
    ref_fn, why = reference_fn()
    results = []
    for name in a.cases:
        c = CASES[name]
        pred, gt = synthetic_pair(c["shape"], c["C"], c["seed"], device="cuda")
        sp = torch.tensor(c["spacing"], dtype=torch.float64)
        for _ in range(2):
            out = b200seg.calculate_distance(pred, gt, sp, c["C"])
        times = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = b200seg.calculate_distance(pred, gt, sp, c["C"])
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        r = dict(case=name, shape=c["shape"], classes=c["C"], gpu_ms_median=1e3 * float(np.median(times)),
                 gpu_ms_min=1e3 * min(times), reps=a.reps)
        if ref_fn is None:
            r.update(ref_s="not measured (%s)" % why, agree=None)
        else:
            pc, gc = pred.cpu(), gt.cpu()
            rt = []
            for _ in range(a.ref_reps):
                t0 = time.perf_counter()
                ref = ref_fn(pc, gc, sp, c["C"])
                rt.append(time.perf_counter() - t0)
            r.update(ref_s=float(np.median(rt)), agree=bool(same(out[0], ref[0]) and same(out[1], ref[1])))
        print("%-5s %s C=%2d  GPU %.2f ms (median of %d, min %.2f)  reference CPU %s  outputs agree: %s"
              % (name, "x".join(map(str, c["shape"])), c["C"], r["gpu_ms_median"], a.reps, r["gpu_ms_min"],
                 ("%.2f s" % r["ref_s"]) if isinstance(r["ref_s"], float) else r["ref_s"], r["agree"]))
        print("      ASD %s\n      HD  %s" % (np.round(out[0], 4), np.round(out[1], 4)))
        results.append(r)
    if a.out:
        json.dump({"gpu": gpu_info(), "cpu": cpu_info(), "results": results}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
