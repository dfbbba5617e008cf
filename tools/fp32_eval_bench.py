"""fp32 validation and fp32 training on one H100: b200seg exact fp32, b200seg TF32, and the unmodified reference on cuDNN.

  python tools/fp32_eval_bench.py [--volume D H W] [--reps N] [--train-shape B D H W] [--layer-reps N] [--out FILE]

Two workloads, both the ResUNet of the KiTS configuration (bench.py `resunet_kits_160`: BasicBlock, base 32, 3^3
kernels, 3 classes) with bench.py's seeded weights:
  * validation: sliding-window inference with the reference's schedule (inference/inference3d.py: 128^3 windows, half
    overlap, the last window snapped to the border, softmax averaged), no autocast, on a seeded synthetic volume of a
    validation-like size (default 1 x 1 x 160 x 256 x 256);
  * training: one fp32 step (forward, Dice + CE, backward, AdamW, EMA), no autocast, at the bench workload's crop.
Three arms, alternated and repeated: b200seg with TF32 off (exact fp32, the CUDA-core convolutions), b200seg with TF32
on (torch.backends.cuda.matmul.fp32_precision = 'tf32'), and the unmodified reference modules from oracle/_ref on stock
PyTorch with default flags, under which cuDNN runs fp32 convolutions on TF32.  Each arm is warmed up, then timed with
CUDA events; median and min over the repeats are reported.  The validation label maps of the arms are compared.

Then a per-layer table: every forward / data-gradient launch of the ResUNet at one 128^3 window, timed with CUDA events
on the CUDA-core kernel (DIRECT) and on the TF32 tensor cores (TC_TF32).  The card's name and power limit are printed
from the same run.  Needs a GPU and oracle/_ref (written by __graft_entry__.build()); there is no fallback."""
import argparse
import json
import os
import statistics
import sys
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import b200seg  # noqa: E402
from b200seg import _lib, ops  # noqa: E402
from layer_times import card, launches  # noqa: E402
from oracle.synth import make_volume  # noqa: E402

WORKLOAD = "resunet_kits_160"
ARMS = ("b200seg_exact", "b200seg_tf32", "reference_cudnn")


def set_tf32(on, saved):
    torch.backends.cuda.matmul.fp32_precision = "tf32" if on else saved


def ref_sliding_window(net, img, window, classes):
    """inference/inference3d.py's schedule, restated in stock PyTorch for the reference arm"""
    B, C, D, H, W = img.shape
    half = [w // 2 for w in window]
    out = torch.zeros(B, classes, D, H, W, device=img.device)
    cnt = torch.zeros(B, 1, D, H, W, device=img.device)

    def split(h, size, i):
        s = h * i
        return (size - 2 * h, size) if s + 2 * h > size else (s, s + 2 * h)
    net.eval()
    with torch.no_grad():
        for i in range(D // half[0]):
            for j in range(H // half[1]):
                for k in range(W // half[2]):
                    (d0, d1), (h0, h1), (w0, w1) = split(half[0], D, i), split(half[1], H, j), split(half[2], W, k)
                    out[:, :, d0:d1, h0:h1, w0:w1] += F.softmax(net(img[:, :, d0:d1, h0:h1, w0:w1]), dim=1)
                    cnt[:, :, d0:d1, h0:h1, w0:w1] += 1
    return out / cnt


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def summary(ts):
    return {"median_ms": statistics.median(ts), "min_ms": min(ts), "runs": len(ts)}


def layer_table(wl, window, reps, saved):
    """[(kind, layer, calls, direct us, tf32 us)] for the forward / data-gradient launches of one window"""
    wl1 = wl[:4] + ((1,) + tuple(window),)
    rows = []
    for kind, ci, co, k, dims, n in launches(wl1):
        x = torch.randn(1, *dims, ci, device="cuda")
        st = ops.instnorm_stats(x, 0, ci)
        w = torch.randn(co, ci, *k, device="cuda") * (2.0 / (ci * k[0] * k[1] * k[2])) ** 0.5
        gx = torch.randn(1, *dims, co, device="cuda") if kind == "dgrad" else None
        gst = ops.instnorm_stats(gx, 0, co) if gx is not None else None
        r = torch.randn(1, *dims, co, device="cuda") if kind == "fwd_res" else None
        t = {}
        for algo in (_lib.ALGO_DIRECT, _lib.ALGO_TC_TF32):
            wp = ops.pack_weight(w, torch.float32, layout=algo)
            if kind == "dgrad":
                fn = lambda: ops.conv3d_fwd(x, 0, ci, None, ops.ACT_NONE, wp, co, k, dgrad_of=(gx, 0, gst, ops.ACT_RELU), algo=algo)
            else:
                fn = lambda: ops.conv3d_fwd(x, 0, ci, st, ops.ACT_RELU, wp, co, k, residual=r, algo=algo)
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            t[algo] = timed(lambda: [fn() for _ in range(reps)])[0] / reps * 1e3
        rows.append((kind, "%d->%d k%s @%s" % (ci, co, "".join(map(str, k)), "x".join(map(str, dims))), n,
                     t[_lib.ALGO_DIRECT], t[_lib.ALGO_TC_TF32]))
        del x, w, gx, r
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--volume", type=int, nargs=3, default=[160, 256, 256])
    ap.add_argument("--window", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--train-shape", type=int, nargs=4, default=None, help="B D H W (default: the bench workload's crop)")
    ap.add_argument("--train-reps", type=int, default=5)
    ap.add_argument("--layer-reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fp32_eval_bench needs a GPU"
    saved = torch.backends.cuda.matmul.fp32_precision
    assert saved != "tf32", "start with TF32 off: the exact arm must be exact"
    wl = bench.WORKLOADS[WORKLOAD]
    scale, kernel, classes, ce_w, crop = wl
    ref = bench.reference_net(wl)
    assert ref is not None, "the reference modules are missing from oracle/_ref: run __graft_entry__.build() first"
    ref_net, ref_loss = ref
    dev = torch.device("cuda")
    info = {"card": card(), "workload": WORKLOAD, "cudnn_conv_fp32_precision": torch.backends.cudnn.conv.fp32_precision}
    print("fp32 validation / training, %s: %s" % (WORKLOAD, info["card"]))

    def ours_net():
        n = b200seg.UNet(1, bench.BASE, scale=scale, kernel_size=kernel, num_classes=classes, block="BasicBlock", norm="in")
        n.load_state_dict(bench.oracle_state(wl))
        return n.to(dev)

    # ---- validation
    D, H, W = args.volume
    img, _ = make_volume(1, D, H, W, classes, seed=2025)
    img = img.to(dev)
    window = [args.window] * 3
    net = ours_net().eval()
    ref_net = ref_net.to(dev).eval()
    ns = types.SimpleNamespace(window_size=window, classes=classes, dimension="3d", sliding_window=True)

    def val(arm):
        set_tf32(arm == "b200seg_tf32", saved)
        if arm == "reference_cudnn":
            return ref_sliding_window(ref_net, img, window, classes).argmax(1)
        return b200seg.inference_sliding_window(net, img, ns, return_label=True)[1].long()
    labels, vt = {}, {a: [] for a in ARMS}
    for a in ARMS:                                          # warm-up (module loads, cuDNN algorithm choice)
        labels[a] = val(a)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for a in ARMS:
            vt[a].append(timed(lambda: val(a))[0])
    set_tf32(False, saved)
    nvox = labels["b200seg_exact"].numel()
    info["validation"] = {
        "volume": [1, 1, D, H, W], "window": window, "windows": (D // (window[0] // 2)) * (H // (window[1] // 2)) * (W // (window[2] // 2)),
        **{a: summary(vt[a]) for a in ARMS},
        "label_agreement_tf32_vs_exact": (labels["b200seg_tf32"] == labels["b200seg_exact"]).sum().item() / nvox,
        "label_agreement_reference_vs_exact": (labels["reference_cudnn"] == labels["b200seg_exact"]).sum().item() / nvox}
    del labels, net
    torch.cuda.empty_cache()

    # ---- one fp32 training step
    from b200seg.train import TrainStep
    B, TD, TH, TW = args.train_shape or crop
    timg, tlab = make_volume(B, TD, TH, TW, classes, seed=2026)
    timg, tlab = timg.to(dev), tlab.to(dev)
    w = torch.tensor(ce_w, device=dev)
    net, ema = ours_net(), ours_net()
    step = TrainStep(net.train(), ema, ce_weight=w.cpu(), amp=False)
    ref_net.train()
    params = list(ref_net.parameters())
    ref_ema = [v.detach().clone() for v in params]
    ce = nn.CrossEntropyLoss(weight=w)
    opt = torch.optim.AdamW(params, lr=1e-3, betas=(0.9, 0.999), weight_decay=0.05, eps=1e-5, fused=True)

    def ref_step():
        opt.zero_grad(set_to_none=True)
        loss = ref_loss(ref_net(timg), tlab, ce)
        loss.backward()
        opt.step()
        torch._foreach_mul_(ref_ema, 0.99)
        torch._foreach_add_(ref_ema, [v.detach() for v in params], alpha=0.01)
        return loss.detach()

    def train(arm):
        set_tf32(arm == "b200seg_tf32", saved)
        return ref_step() if arm == "reference_cudnn" else step(timg, tlab)
    tt, losses = {a: [] for a in ARMS}, {}
    for a in ARMS:
        for _ in range(2):
            train(a)
    torch.cuda.synchronize()
    for _ in range(args.train_reps):
        for a in ARMS:
            t, loss = timed(lambda: train(a))
            tt[a].append(t)
            losses[a] = loss.item()
    set_tf32(False, saved)
    info["train_step"] = {"shape": [B, 1, TD, TH, TW], **{a: summary(tt[a]) for a in ARMS}, "last_loss": losses}
    del net, ema, step, opt, ref_ema, params
    ref_net.cpu()
    torch.cuda.empty_cache()

    # ---- per-layer table at one validation window
    rows = layer_table(wl, window, args.layer_reps, saved)
    info["layers"] = [dict(kind=k, layer=l, calls=n, direct_us=d, tf32_us=t) for k, l, n, d, t in rows]

    for name in ("validation", "train_step"):
        r = info[name]
        print("%-10s %s: %s" % (name, r.get("volume", r.get("shape")),
                                ", ".join("%s %.1f ms (min %.1f)" % (a, r[a]["median_ms"], r[a]["min_ms"]) for a in ARMS)))
    print("validation label agreement with the exact path: TF32 %.6f, reference on cuDNN %.6f"
          % (info["validation"]["label_agreement_tf32_vs_exact"], info["validation"]["label_agreement_reference_vs_exact"]))
    print("%-8s %-32s %5s | %10s %10s %7s" % ("kind", "layer", "calls", "DIRECT us", "TF32 us", "speedup"))
    for k, l, n, d, t in rows:
        print("%-8s %-32s %5d | %10.1f %10.1f %7.2f" % (k, l, n, d, t, d / t))
    line = json.dumps(info)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
