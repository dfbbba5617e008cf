"""Per-layer timing of the tensor-core weight gradient (b200seg_conv3d_wgrad) on every distinct weight-gradient call of
one bench.py training step, fused conv1|shortcut shapes included.

  python tools/wgrad_layers.py [--workload NAME] [--reps N] [--json FILE]

Runs one training step of the workload with ops.conv3d_wgrad wrapped to record each call's shape, operand layout
(ld / channel offset) and input transform, then times each distinct call with CUDA events: the C entry point back to
back into preallocated dW / workspace, the split-K slice sum included.  Per shape it prints the calls per step, the
kernel's job split (jobs, split-K factor S, CTAs), its ring (stages NS; whole 16x8 tiles or 8-row halves), the staged
image of x and dy (r32 / r64: swizzled rows of 32 / 64 channels per voxel, p8: 16-byte channel planes), the bytes and
TMA lines (one innermost box row each) the kernel stages into shared memory per call (computed from the shape), the
time, TFLOP/s, the staged rate per CTA, and the FLOP-weighted sum per step.  The launch configuration is the host-side choice of csrc/wgrad_tc.cu (pick_ntc / fill_params), mirrored
here.  The card name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

NUM_SMS, MT, MAX_COLS, MAX_STAGES = 132, 128, 192, 6
SMEM = 227 * 1024 - 2048


def pick_ntc(cin):
    if cin % 16:
        return 0
    if cin % 128 == 0:
        return 64
    if cin <= 128:
        return cin
    return next((v for v in (128, 96, 64, 48, 32, 16) if cin % v == 0), 0)


def plan(cin, cout, k, B, D, H, W):
    """fill_params of csrc/wgrad_tc.cu: job split, split-K factor, ring, staged bytes per call; None if not on the
    tensor cores by shape"""
    kd, kh, kw = k
    ntc = pick_ntc(cin)
    if not ntc or cout % 8 or B * ntc > 2048 or max(k) > 3:
        return None
    taps_hw = kh * kw
    g = min(MAX_COLS // ntc, taps_hw)
    ngroups = -(-taps_hw // g)
    co_max = min(cout, MT)

    def ring(ts, dy_ch, x_ch):
        rows = dy_ch != 8 or x_ch != 8
        halo_w, halo_h = 8 + kw - 1, ts + kh - 1
        a_group = halo_h * halo_w * x_ch * 2
        if x_ch == 32:
            a_group = -(-a_group // 512) * 512
        align = 1024 if rows else 128
        a_box = ntc * halo_h * halo_w * 2
        dy_box = co_max * ts * 8 * 2
        stage = -(-(ntc // x_ch * a_group) // align) * align + dy_box
        tail = max(0, -(-co_max // 64) * 8 * ts * 8 * 16 - stage) if dy_ch == 8 else 0
        lines = halo_h * halo_w * (ntc // x_ch) + ts * 8 * (co_max // dy_ch)
        return min((SMEM - tail - B * ntc * 8) // stage, MAX_STAGES), a_box + dy_box, lines

    def size(dy_ch, x_ch):
        ts = 16
        r = ring(ts, dy_ch, x_ch)
        if r[0] < 4:
            ts = 8
            r = ring(ts, dy_ch, x_ch)
        return (ts, dy_ch, x_ch) + r

    # row images unless they cost the ring a stage (a row image next to a plane image)
    planes = size(8, 8)
    dy_ch = 32 if co_max == 32 else 64 if (co_max == 64 or (co_max == MT and cout % 64 == 0)) else 8
    x_ch = 64 if ntc == 64 else 32 if ntc in (32, 96) else 8
    pick = size(dy_ch, x_ch)
    if pick[:4:3] != planes[:4:3]:
        pick = planes
    ts, dy_ch, x_ch, ns, stage_tx, stage_lines = pick
    if ns < 2:
        return None
    tiles_hw = -(-H // 16) * -(-W // 8)
    jobs = -(-cout // MT) * (cin // ntc) * kd * ngroups
    S = min(max(1, NUM_SMS // jobs), B * D * tiles_hw)
    # every job stages each voxel tile whose input depth slice lies inside the volume, in 16 / ts stages
    valid_tiles = sum(B * max(0, min(D, D - (zd - kd // 2)) - max(0, -(zd - kd // 2))) * tiles_hw for zd in range(kd))
    stages = -(-cout // MT) * (cin // ntc) * ngroups * valid_tiles * (16 // ts)
    image = "%s/%s" % ("p8" if x_ch == 8 else "r%d" % x_ch, "p8" if dy_ch == 8 else "r%d" % dy_ch)
    return dict(jobs=jobs, S=S, ctas=jobs * S, NS=ns, staging="half" if ts == 8 else "whole", image=image,
                staged=stages * stage_tx, lines=stages * stage_lines)


def record_calls(workload):
    """(key -> calls per step) of one training step; key = the arguments that fix what the kernel does"""
    import torch
    import b200seg
    from b200seg import ops
    from b200seg.train import TrainStep
    from oracle.synth import make_volume

    wl = bench.WORKLOADS[workload]
    assert not bench.is_swin(wl) and not bench.is_medformer(wl), "the ResUNet workloads only"
    scale, kernel, classes, weight, (B, D, H, W) = wl
    dev = torch.device("cuda", 0)

    def make_net():
        n = b200seg.UNet(1, bench.BASE, scale=scale, kernel_size=kernel, num_classes=classes, block="BasicBlock", norm="in")
        n.load_state_dict(bench.oracle_state(wl))
        return n.to(dev)

    net, ema = make_net(), make_net()
    for p in ema.parameters():
        p.requires_grad_(False)
    ts = TrainStep(net, ema, ce_weight=torch.tensor(weight), amp=True)
    img, lab = make_volume(B, D, H, W, classes, seed=2023)
    img, lab = img.to(dev), lab.to(dev)
    ts(img, lab)                                   # warm-up: weight packing, workspaces
    calls = {}
    inner = ops.conv3d_wgrad

    def wrapped(x, x_coff, Cin, x_stats, act, dy, dy_coff, Cout, ksize, want_bias=False, algo=ops.ALGO_AUTO, eps=ops.IN_EPS):
        key = (tuple(x.shape), x_coff, Cin, x_stats is not None, act, dy.shape[-1], dy_coff, Cout, tuple(ksize),
               bool(want_bias), algo, x.dtype == torch.float16)
        calls[key] = calls.get(key, 0) + 1
        return inner(x, x_coff, Cin, x_stats, act, dy, dy_coff, Cout, ksize, want_bias, algo, eps)

    ops.conv3d_wgrad = wrapped
    try:
        ts(img, lab)
        torch.cuda.synchronize()
    finally:
        ops.conv3d_wgrad = inner
    del net, ema, ts
    return calls


def time_call(key, reps):
    import torch
    from b200seg import _lib, ops
    (B, D, H, W, x_ld), x_coff, Cin, stats, act, dy_ld, dy_coff, Cout, k, want_bias, algo, f16 = key
    dt = torch.float16 if f16 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, D, H, W, x_ld, device="cuda", generator=g).to(dt)
    dy = torch.randn(B, D, H, W, dy_ld, device="cuda", generator=g).to(dt)
    st = ops.instnorm_stats(x, x_coff, Cin) if stats else None
    dw = torch.zeros(Cout, Cin, *k, device="cuda")
    db = torch.zeros(Cout, device="cuda") if want_bias else None
    lib = _lib.load()
    ws_bytes = lib.b200seg_conv3d_wgrad_workspace(x_ld, x_coff, 1 if (stats or act) else 0, dy_ld, dy_coff, 1 if want_bias else 0,
                                                  B, D, H, W, Cin, Cout, *k, ops._dt(x), algo)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")

    def run():
        _lib.call("b200seg_conv3d_wgrad", x.data_ptr(), x_ld, x_coff, ops._p(st), ops.IN_EPS, act, dy.data_ptr(), dy_ld, dy_coff,
                  dw.data_ptr(), ops._p(db), B, D, H, W, Cin, Cout, *k, ops._dt(x), algo, ws.data_ptr() if ws_bytes else None,
                  ws_bytes, ops._stream())

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="resunet_acdc_128", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    import torch
    from b200seg import _lib
    assert torch.cuda.is_available(), "wgrad_layers needs a GPU"
    torch.cuda.set_device(0)
    assert _lib.load().b200seg_check_device() == 0, "not an sm_90 device"

    name, power = card()
    calls = record_calls(args.workload)
    rows = []
    for key, n in sorted(calls.items(), key=lambda kv: (kv[0][7], kv[0][2], kv[0][0])):
        (B, D, H, W, x_ld), x_coff, Cin, stats, act, _, _, Cout, k, _, _, _ = key
        pl = plan(Cin, Cout, k, B, D, H, W) or {}
        us = time_call(key, args.reps)
        flop = 2.0 * B * D * H * W * Cin * Cout * k[0] * k[1] * k[2]
        rows.append(dict(shape="%d->%d k%s @%dx%dx%dx%d" % (Cin, Cout, "".join(map(str, k)), B, D, H, W),
                         x_layout="%d+%d" % (x_ld, x_coff),
                         xform="IN+act" if stats else ("act" if act else "raw"), calls=n, us=us, tflops=flop / us / 1e6,
                         flop=flop, **pl))
    total_us = sum(r["us"] * r["calls"] for r in rows)
    total_flop = sum(r["flop"] * r["calls"] for r in rows)
    print("workload %s on %s, power limit %s" % (args.workload, name, power))
    hdr = "%-28s %-7s %-6s %5s %5s %3s %5s %2s %-5s %-7s %9s %8s %9s %8s %9s" % (
        "layer", "x ld+c0", "input", "calls", "jobs", "S", "CTAs", "NS", "tile", "x/dy", "MB staged", "M lines", "us", "TFLOP/s",
        "GB/s/CTA")
    print(hdr)
    for r in rows:
        per_cta = "%.1f" % (r["staged"] / r["us"] / 1e3 / r["ctas"]) if "staged" in r else "-"
        print("%-28s %-7s %-6s %5d %5s %3s %5s %2s %-5s %-7s %9s %8s %9.1f %8.1f %9s" % (
            r["shape"], r["x_layout"], r["xform"], r["calls"], r.get("jobs", "-"), r.get("S", "-"), r.get("ctas", "-"), r.get("NS", "-"),
            r.get("staging", "-"), r.get("image", "-"), "%.1f" % (r["staged"] / 1e6) if "staged" in r else "-",
            "%.2f" % (r["lines"] / 1e6) if "lines" in r else "-", r["us"], r["tflops"], per_cta))
    print("per step: %d calls, %.3f ms, %.1f GFLOP, %.1f TFLOP/s (FLOP-weighted)" % (
        sum(r["calls"] for r in rows), total_us / 1e3, total_flop / 1e9, total_flop / total_us / 1e6))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(workload=args.workload, card=name, power_limit=power, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
