"""Where the time of one bench.py training step goes: device time per kernel, summed over the profiled steps.

  python tools/step_profile.py --out DIR [--workload NAME] [--steps K] [--warmup W]

Builds the same model, TrainStep and synthetic volume as bench.py, runs W untimed steps, then K steps under
torch.profiler with CUDA activities.  Writes DIR/trace.json (Chrome trace) and DIR/kernels.txt: per kernel name the
device time per step, its share of the summed kernel time, and the launches per step, followed by the step's wall time
(CUDA events, profiler running) and the gap between it and the summed kernel time (launch gaps, host stalls).  Kernels
are grouped by their name without template arguments, so every instantiation of a kernel template is one row.
Run it on its own: the profiler slows the host, so its wall time is not the bench.py number."""
import argparse
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def kernel_group(name):
    """'void (anonymous namespace)::conv_tc_kernel<128, 4>((anonymous namespace)::TcParams)' -> 'conv_tc_kernel'"""
    s = name.replace("(anonymous namespace)::", "")
    if s.startswith("void "):
        s = s[5:]
    s = re.split(r"[<(]", s, maxsplit=1)[0].strip()
    return s.split("::")[-1] or name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="resunet_acdc_128", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True, help="directory for trace.json and kernels.txt")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import b200seg
    from b200seg import _lib
    from b200seg.train import TrainStep
    from oracle.synth import make_volume

    wl = bench.WORKLOADS[args.workload]
    scale, kernel, classes, weight, (B, D, H, W) = wl
    med = bench.is_medformer(wl)
    assert torch.cuda.is_available(), "step_profile needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    assert _lib.load().b200seg_check_device() == 0, "not an sm_90 device"

    def make_net():                               # the models bench.run_b200 builds
        if bench.is_swin(wl):
            n = b200seg.SwinUNETR((D, H, W), 1, classes, feature_size=wl[1])
            n.load_state_dict(bench.oracle_state(wl), strict=False)
            return n.to(dev)
        if med:
            n = b200seg.MedFormer(1, classes, bench.BASE, conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0,
                                  proj_type="depthwise", norm="in", act="relu", **wl[0])
        else:
            n = b200seg.UNet(1, bench.BASE, scale=scale, kernel_size=kernel, num_classes=classes, block="BasicBlock", norm="in")
        n.load_state_dict(bench.oracle_state(wl))
        return n.to(dev)

    net, ema = make_net(), make_net()
    for p in ema.parameters():
        p.requires_grad_(False)
    ts = TrainStep(net, ema, ce_weight=torch.tensor(weight), amp=True, aux_weight=bench.AUX_WEIGHT if med else None)
    img, lab = make_volume(B, D, H, W, classes, seed=2023)
    img, lab = img.to(dev), lab.to(dev)

    for _ in range(max(args.warmup, 1)):
        ts(img, lab)
    torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0.record()
        for _ in range(args.steps):
            ts(img, lab)
        e1.record()
        torch.cuda.synchronize()
    wall_ms = e0.elapsed_time(e1) / args.steps
    prof.export_chrome_trace(os.path.join(args.out, "trace.json"))

    groups = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        dt = getattr(ev, "device_time", None)
        if dt is None:
            dt = ev.cuda_time
        if not dt:
            continue
        g = groups.setdefault(kernel_group(ev.name), [0.0, 0])
        g[0] += dt / 1e3                           # us -> ms
        g[1] += 1
    total = sum(v[0] for v in groups.values()) / args.steps
    name = torch.cuda.get_device_name(dev)
    lines = ["workload %s, %d profiled steps on %s" % (args.workload, args.steps, name),
             "%-44s %12s %8s %10s" % ("kernel", "ms/step", "share", "launches")]
    for k, (t, n) in sorted(groups.items(), key=lambda kv: -kv[1][0]):
        lines.append("%-44s %12.3f %7.1f%% %10.1f" % (k[:44], t / args.steps, 100.0 * t / args.steps / total, n / args.steps))
    lines += ["%-44s %12.3f" % ("sum of kernel time", total),
              "%-44s %12.3f" % ("step wall time (CUDA events, profiler on)", wall_ms),
              "%-44s %12.3f %7.1f%%" % ("gap (wall - kernels)", wall_ms - total, 100.0 * (wall_ms - total) / wall_ms)]
    text = "\n".join(lines)
    with open(os.path.join(args.out, "kernels.txt"), "w") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
