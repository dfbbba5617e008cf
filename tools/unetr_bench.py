#!/usr/bin/env python
"""unetr_bench.py — training-step time of UNETR at the bcv configuration (get_model: 96^3 crop, 14 classes, ViT-B/16,
feature_size 16) on one GPU, for b200seg and for a stock-PyTorch arm.

  python tools/unetr_bench.py [--batch 1 2] [--steps 20] [--warmup 5] [--profile DIR]

One step = zero_grad -> autocast fp16 forward -> CE + Dice -> scaled backward -> fused AdamW -> EMA, as bench.py times
the other models.
  b200seg : b200seg.get_model(args) driven by b200seg.train.TrainStep (FusedAdamWEMA).
  stock   : oracle/unetr.py (UNETR as a function of its state_dict, the same algorithm) under stock torch autocast +
            cuDNN (benchmark mode), torch's fused AdamW, GradScaler and a foreach EMA.  The reference class itself
            cannot be imported without monai, so — as bench.py does for SwinUNETR — the oracle stands in for it.
Both arms are timed with CUDA events over --steps steps after --warmup steps; the GPU name, power limit and the SM
clocks sampled during the timed loops are printed beside each number.
--profile DIR instead runs a few b200seg steps under torch.profiler and writes DIR/unetr_profile_b<B>.txt: the kernel table,
the attention kernels' share of the step's device time, and the ViT GEMMs' share.  The same GEMM kernels also run the
decoder's convolutions, so kernel names alone cannot separate them: the ViT GEMM time is taken from a second profile of
the ViT alone (forward + backward of the same model), where every convolution-family kernel is a ViT Linear."""
import argparse
import json
import os
import re
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import ClockSampler     # noqa: E402

CLASSES, SIZE = 14, (96, 96, 96)
CE_W = [0.5] + [1.0] * 13
ATTN = re.compile(r"attn_(fwd|bwd|delta)")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, mx = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": plim, "sm_max_clock": mx}
    except Exception as e:                 # the numbers are printed anyway; say why the card is unknown
        return {"gpu": "unknown (%s)" % e}


def setup(B, seed=7):
    import torch
    import b200seg
    from oracle import unetr as ounetr
    from oracle.synth import make_volume
    shapes = ounetr.unetr_param_shapes(1, CLASSES, SIZE)
    sd = ounetr.seeded_state_dict(shapes, seed)
    img, lab = make_volume(B, *SIZE, CLASSES, seed=2024)
    args = types.SimpleNamespace(dimension="3d", model="unetr", in_chan=1, classes=CLASSES, training_size=list(SIZE))
    return torch, b200seg, ounetr, sd, img.cuda(), lab.cuda(), args


def b200_step(B):
    torch, b200seg, _, sd, img, lab, args = setup(B)
    from b200seg.train import TrainStep
    net = b200seg.get_model(args)
    net.load_state_dict(sd)
    ema = b200seg.get_model(args)
    ema.load_state_dict(sd)
    step = TrainStep(net.cuda(), ema.cuda(), ce_weight=torch.tensor(CE_W), amp=True)
    return torch, (lambda: step(img, lab)), net


def stock_step(B):
    torch, _, ounetr, sd, img, lab, _ = setup(B)
    from oracle import losses as olosses
    torch.backends.cudnn.benchmark = True
    params = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
    plist = list(params.values())
    ema = [p.detach().clone() for p in plist]
    opt = torch.optim.AdamW(plist, lr=1e-3, betas=(0.9, 0.999), weight_decay=0.05, eps=1e-5, fused=True)
    scaler = torch.amp.GradScaler("cuda")
    w = torch.tensor(CE_W, device="cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            loss = olosses.total_loss(ounetr.unetr_forward(params, img, 12), lab, w)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        torch._foreach_mul_(ema, 0.99)
        torch._foreach_add_(ema, [p.detach() for p in plist], alpha=0.01)
        return loss.detach()
    return torch, step, None


def timed(torch, step, warmup, steps, cs):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with cs.window():
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def vit_profile(torch, net, img, n):
    """the ViT alone, forward + backward (gradients into the four outputs the decoder reads), under torch.profiler:
    every convolution-family kernel of this run is a ViT Linear"""
    from torch.profiler import ProfilerActivity, profile as tprof
    x = img.permute(0, 2, 3, 4, 1).half().contiguous()

    def run():
        with torch.autocast("cuda", dtype=torch.float16):
            net._packs.refresh()
            last, hs = net.vit(x)
        outs = [last, hs[3], hs[6], hs[9]]
        torch.autograd.backward(outs, [torch.ones_like(o) * 1e-3 for o in outs])
    run()
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            run()
        torch.cuda.synchronize()
    gemm = re.compile(r"conv_tc_kernel|wgrad_tc_kernel|bias_grad_kernel|add_slices|conv_fwd_direct")
    return sum(e.self_device_time_total for e in prof.key_averages()
               if e.device_type.name == "CUDA" and gemm.search(e.key)) / n / 1e3


def profile(out_dir, B, warmup):
    from torch.profiler import ProfilerActivity, profile as tprof
    torch, step, net = b200_step(B)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    n = 3
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    rows = [e for e in prof.key_averages() if e.device_type.name == "CUDA"]
    total = sum(e.self_device_time_total for e in rows) / n / 1e3
    attn = sum(e.self_device_time_total for e in rows if ATTN.search(e.key)) / n / 1e3
    _, _, _, _, img, _, _ = setup(B)
    vit = vit_profile(torch, net, img, n)
    info = gpu_info()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "unetr_profile_b%d.txt" % B)
    with open(path, "w") as f:
        f.write("UNETR bcv 96^3 B=%d, AMP training step (b200seg), %s, power limit %s\n" % (B, info.get("gpu"), info.get("power_limit")))
        f.write("device time per step (sum of kernels) %.2f ms\n" % total)
        f.write("attention kernels (attn_*): %.3f ms = %.1f %%\n" % (attn, 100 * attn / total))
        f.write("ViT GEMMs (fwd + bwd of the 49 ViT Linears, from a profile of the ViT alone): %.2f ms = %.1f %%\n"
                % (vit, 100 * vit / total))
        f.write(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=30))
    print(json.dumps({"profile": path, "batch": B, "device_ms_per_step": round(total, 3), "attention_ms": round(attn, 3),
                      "attention_share": round(attn / total, 4), "vit_gemm_ms": round(vit, 3),
                      "vit_gemm_share": round(vit / total, 4), **info}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", metavar="DIR")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("unetr_bench.py measures on a CUDA device; none is available")
    if a.profile:
        for B in a.batch:
            profile(a.profile, B, a.warmup)
        return
    info = gpu_info()
    for B in a.batch:
        for arm, make in (("b200seg", b200_step), ("stock", stock_step)):
            torch, step, _ = make(B)
            with ClockSampler(0) as cs:
                ms = timed(torch, step, a.warmup, a.steps, cs)
            vox = B * SIZE[0] * SIZE[1] * SIZE[2]
            print(json.dumps({"model": "unetr_bcv_96", "arm": arm, "batch": B, "ms_per_step": round(ms, 3),
                              "voxels_per_s": round(vox / ms * 1e3), "steps": a.steps, "clocks": cs.summary(), **info}))
            del step
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
