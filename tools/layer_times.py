"""Per-launch timing of the tensor-core forward / data-gradient convolution (`conv_tc_kernel`) on the exact launches of
one training step of a bench.py ResUNet workload, CUDA events, C entry points called back to back.

  python tools/layer_times.py [--workload NAME] [--reps N]

The launches are derived from `bench.conv_layers()`: per BasicBlock the fused conv1|shortcut forward (IN+ReLU loader,
no side operand), the conv2 forward (IN+ReLU loader + residual epilogue), and the two data-gradient launches (dy ->
dx with the InstanceNorm/ReLU mask of the saved input, `gx`, in the epilogue).  Each row also times the conv2 shape
without its residual, so the cost of the side operand can be read off.  Per row: time, TFLOP/s, the HBM floor (the
bytes every operand must cross once, over 3.35 TB/s, the H100 SXM data-sheet bandwidth) and floor / time; the last
line sums the rows over one step."""
import argparse
import os
import subprocess
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from b200seg import ops  # noqa: E402

HBM_BPS = 3.35e12


def launches(wl):
    """[(kind, Cin, Cout, k, dims, calls per step)] of conv_tc_kernel, kind in fwd / fwd_res / dgrad"""
    scale, kernel, classes, _, (B, D, H, W) = wl
    L = [(ci, co, tuple(k), d) for ci, co, k, d in bench.conv_layers(scale, kernel, classes, B, D, H, W)]
    out = {}

    def add(key):
        out[key] = out.get(key, 0) + 1
    i = 0
    while i < len(L):
        ci, co, k, d = L[i]
        if ci % 16 or co % 16:                       # stem (Cin 1) and the 1x1x1 head take other kernels
            i += 1
            continue
        fused = i + 2 < len(L) and L[i + 2] == L[i] and ci != co
        cf = 2 * co if fused else co
        add(("fwd", ci, cf, k, d)); add(("fwd_res", co, co, k, d))
        add(("dgrad", co, co, k, d)); add(("dgrad", cf, ci, k, d))
        i += 3 if fused else 2
    return [(kind, ci, co, k, d, n) for (kind, ci, co, k, d), n in out.items()]


def hbm_bytes(kind, ci, co, k, vox):
    w = ci * co * k[0] * k[1] * k[2] * 2
    act = {"fwd": ci + co, "fwd_res": ci + 2 * co, "dgrad": ci + 2 * co}[kind]
    return vox * act * 2 + w


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "power limit unknown"
    return "%s, %s" % (name, q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="resunet_acdc_128",
                    choices=[k for k, v in bench.WORKLOADS.items() if not bench.is_medformer(v) and not bench.is_swin(v)])
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "layer_times needs a GPU"
    wl = bench.WORKLOADS[args.workload]
    B = wl[4][0]
    torch.manual_seed(0)

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps * 1e3

    print("%s, %s" % (args.workload, card()))
    hdr = "%-8s %-30s %5s | %9s %7s %9s %6s | %13s" % ("kind", "layer", "calls", "us", "TFLOP/s", "floor us", "floor",
                                                        "us w/o side")
    print(hdr)
    tot = [0.0, 0.0]
    for kind, ci, co, k, (D, H, W), n in launches(wl):
        vox = B * D * H * W
        x = torch.randn(B, D, H, W, ci, device="cuda").half()
        st = ops.instnorm_stats(x, 0, ci)
        w = torch.randn(co, ci, *k, device="cuda") * 0.05
        algo = ops.conv_algo(ci, co, k, torch.float16, B)
        wp = (ops.pack_weight(w, torch.float16, layout=algo), algo)
        side_free = None
        if kind == "dgrad":                          # dy = x (raw), dx has co channels, gx the saved forward input
            gx = torch.randn(B, D, H, W, co, device="cuda").half()
            gst = ops.instnorm_stats(gx, 0, co)
            t = timed(lambda: ops.conv3d_fwd(x, 0, ci, None, ops.ACT_NONE, wp, co, k, dgrad_of=(gx, 0, gst, ops.ACT_RELU)))
            del gx
        else:
            r = torch.randn(B, D, H, W, co, device="cuda").half() if kind == "fwd_res" else None
            t = timed(lambda: ops.conv3d_fwd(x, 0, ci, st, ops.ACT_RELU, wp, co, k, residual=r))
            if r is not None:
                side_free = timed(lambda: ops.conv3d_fwd(x, 0, ci, st, ops.ACT_RELU, wp, co, k))
            del r
        fl = 2.0 * vox * ci * co * k[0] * k[1] * k[2]
        floor = hbm_bytes(kind, ci, co, k, vox) / HBM_BPS * 1e6
        tot[0] += n * t; tot[1] += n * floor
        print("%-8s %-30s %5d | %9.1f %7.1f %9.1f %6.2f | %13s" % (
            kind, "%d->%d k%s @%dx%s" % (ci, co, "".join(map(str, k)), B, "x".join(map(str, (D, H, W)))), n,
            t, fl / (t * 1e-6) / 1e12, floor, floor / t, "%.1f" % side_free if side_free is not None else "-"))
        del x, w
    print("per step: %.2f ms in conv_tc_kernel, HBM floor %.2f ms (%.2f)" % (tot[0] / 1e3, tot[1] / 1e3, tot[1] / tot[0]))


if __name__ == "__main__":
    main()
