"""Time the ACDC 2D training augmentation (dataset_acdc.py:128-142) for one batch of 32 slices, four ways, in one run:
  * b200seg.augmentation.TrainAugment2D — plan (host draws) + one table upload + three launches, then apply() with
    the plans made, then the three launches alone (events around the call, and device time from torch.profiler);
  * the same branch through the public per-function GPU path (5 calls per slice) and a stack into [B, 1, h, w];
  * the UNMODIFIED reference functions (oracle/_ref, training/augmentation.py) on the GPU with stock torch;
  * the same reference functions on the host CPU, per slice, single-threaded (the reference runs them in DataLoader
    workers; the 4-worker per-batch figure is derived from the single-thread one, not measured).
Slice sizes are an assumption: the ACDC dataset pads every slice to at least training_size + 10, so the batch is drawn
uniformly from 266-300 x 266-340 (seeded).  Each event timing is 5 (reference on the GPU: 3) windows of repeated calls
after warm-up, reported as median / min / max.  Prints one JSON object with the card name and power limit.
Usage (on the GPU):  python tools/aug2d_bench.py"""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from b200seg import augmentation as aug           # noqa: E402
from oracle import augmentation2d as o2           # noqa: E402

B, SIZE = 32, [256, 256]
H_RANGE, W_RANGE = (266, 301), (266, 341)
ACDC = dict(scale=0.3, rotate=180, translate=0, gaussian_noise_std=0.02, additive_brightness_std=0.7, gamma_range=[0.5, 1.6])


def timed(fn, iters=20, warm=3, repeats=5):
    """CUDA events around `iters` calls after `warm` untimed ones, `repeats` times: (median, min, max) ms per call."""
    for _ in range(warm):
        fn()
    t = sorted(_window(fn, iters) for _ in range(repeats))
    return {"median": round(t[len(t) // 2], 3), "min": round(t[0], 3), "max": round(t[-1], 3)}


def kernel_ms(fn, iters=20):
    """Device time of the b200seg_aug2d_train kernels alone, per call, from torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if "aug2d_" in e.key:
            name = re.search(r"aug2d_\w+(<[^>]*>)?", e.key).group(0)
            per[name] = per.get(name, 0.0) + (getattr(e, "self_device_time_total", None) or e.self_cuda_time_total)
    return round(sum(per.values()) / iters / 1e3, 3), {k: round(v / iters / 1e3, 3) for k, v in per.items()}


def _window(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters          # ms


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:          # noqa: BLE001 — report, never guess
        info["power_limit"] = "unavailable (%r)" % e
    return info


def main():
    torch.cuda.set_device(0)
    rng = np.random.RandomState(0)
    cpu_imgs, cpu_labs = [], []
    for i in range(B):
        img, lab = o2.make_slice(int(rng.randint(*H_RANGE)), int(rng.randint(*W_RANGE)), 4, seed=1000 + i)
        cpu_imgs.append(img)
        cpu_labs.append(lab)
    imgs = [t.cuda() for t in cpu_imgs]
    labs = [t.cuda() for t in cpu_labs]
    ta = aug.TrainAugment2D(SIZE, **ACDC)
    np.random.seed(1)
    torch.manual_seed(1)
    plans = [ta.plan(t.shape) for t in imgs]
    out = {"what": "ACDC 2D train augmentation, one batch of %d slices -> [%d, 1, %d, %d]" % (B, B, *SIZE),
           "slice_sizes_assumed": "uniform %d-%d x %d-%d (training_size + 10 padding and up), seeded"
                                  % (H_RANGE[0], H_RANGE[1] - 1, W_RANGE[0], W_RANGE[1] - 1),
           "card": card(), "ms_per_batch": {}}
    ms = out["ms_per_batch"]
    ms["TrainAugment2D: plan + table packing + upload + 3 launches"] = timed(lambda: ta(imgs, labs))
    ms["TrainAugment2D.apply, plans made: table packing + upload + 3 launches"] = timed(lambda: ta.apply(imgs, labs, plans))
    launch = ta._prepare(imgs, labs, plans)
    ms["the 3 launches alone, table uploaded (events around the call)"] = timed(launch)

    def per_function():
        oi, ol = [], []
        for x, l in zip(imgs, labs):
            t = aug.gaussian_noise(x[None, None], std=0.02)
            t = aug.brightness_additive(t, std=0.7)
            t = aug.gamma(t, gamma_range=[0.5, 1.6], retain_stats=True)
            t, tl = aug.random_scale_rotate_translate_2d(t, l[None, None], 0.3, 180, 0)
            t, tl = aug.crop_2d(t, tl, SIZE, mode="random")
            oi.append(t)
            ol.append(tl)
        return torch.cat(oi), torch.cat(ol)
    ms["b200seg per-function GPU path"] = timed(per_function, iters=5, warm=2)

    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    try:
        import training.augmentation as ref
    except Exception as e:          # noqa: BLE001 — oracle/_ref absent
        out["reference"] = "unavailable (%r)" % e
        print(json.dumps(out, indent=1))
        return

    def ref_slice(x, l):
        x, l = x[None, None], l[None, None]
        x = ref.gaussian_noise(x, std=0.02)
        x = ref.brightness_additive(x, std=0.7)
        x = ref.gamma(x, gamma_range=[0.5, 1.6], retain_stats=True)
        x, l = ref.random_scale_rotate_translate_2d(x, l, 0.3, 180, 0)
        x, l = ref.crop_2d(x, l, SIZE, mode="random")
        return x.squeeze(0), l.squeeze(0)

    def ref_gpu():
        res = [ref_slice(x, l.long()) for x, l in zip(imgs, labs)]
        return torch.stack([r[0] for r in res]), torch.stack([r[1] for r in res])
    ms["reference functions, GPU, stock torch"] = timed(ref_gpu, iters=5, warm=2, repeats=3)

    torch.set_num_threads(1)
    clabs = [l.long() for l in cpu_labs]
    for x, l in zip(cpu_imgs[:4], clabs[:4]):
        ref_slice(x, l)
    per = []
    for _ in range(5):
        for x, l in zip(cpu_imgs, clabs):
            t0 = time.perf_counter()
            ref_slice(x, l)
            per.append((time.perf_counter() - t0) * 1e3)
    cpu_slice = float(np.mean(per))
    out["reference_cpu_single_thread"] = {"ms_per_slice_mean": round(cpu_slice, 3),
                                          "ms_per_slice_median": round(float(np.median(per)), 3),
                                          "ms_per_batch_one_thread (measured per slice x %d)" % B: round(cpu_slice * B, 2),
                                          "ms_per_batch_4_workers (derived: / 4, not measured)": round(cpu_slice * B / 4, 2)}
    out["reference_cpu_single_thread"]["ms_per_slice_min_max"] = [round(min(per), 3), round(max(per), 3)]
    torch.set_num_threads(os.cpu_count() or 1)
    total, per_kernel = kernel_ms(launch)          # last: the profiler run is its own measurement
    out["kernel_device_ms_per_batch (torch.profiler)"] = {"sum": total, "per_kernel": per_kernel}
    ours = ms["TrainAugment2D: plan + table packing + upload + 3 launches"]["median"]
    out["speedup_vs_reference_gpu"] = round(ms["reference functions, GPU, stock torch"]["median"] / ours, 1)
    out["speedup_vs_reference_cpu_4_workers_derived"] = round(cpu_slice * B / 4 / ours, 1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
