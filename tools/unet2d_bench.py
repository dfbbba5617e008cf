#!/usr/bin/env python
"""unet2d_bench.py — training-step time of the ACDC 2D configurations (config/acdc/unet_2d.yaml, resunet_2d.yaml:
model/dim2/unet.py, base 32, 4 classes, batch 32 of 1x256x256 slices) on one GPU, for b200seg and for stock PyTorch.

  python tools/unet2d_bench.py [--blocks SingleConv BasicBlock] [--batch 32] [--size 256] [--steps 20] [--warmup 5]

One step = zero_grad -> autocast fp16 forward -> CE(weight) + Dice -> scaled backward -> AdamW -> EMA (parameters,
then every buffer copied, training/utils.py:98-105).
  b200seg : b200seg.UNet2D with b200seg.DiceCELoss and b200seg.train.FusedAdamWEMA.
  stock   : oracle/unet2d.py (the reference class restated in stock torch and pinned to it by
            oracle/make_golden_unet2d.py) under torch autocast + cuDNN, torch's fused AdamW, GradScaler and a foreach
            EMA; best of cuDNN default, cudnn.benchmark, and cudnn.benchmark + channels_last.
Both arms are timed with CUDA events over --steps steps after --warmup steps.  Every result line carries the GPU name
and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                   # noqa: E402

import b200seg                                 # noqa: E402
from b200seg.train import FusedAdamWEMA        # noqa: E402
from oracle import losses as olosses           # noqa: E402
from oracle.unet2d import UNet2DRef            # noqa: E402

CE_WEIGHT = [0.5, 1.0, 1.0, 1.0]


def card():
    if not torch.cuda.is_available():
        raise SystemExit("unet2d_bench.py measures on a CUDA device; none is visible")
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return {"gpu": name, "power_limit_w": power}


def data(B, S):
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randn(B, 1, S, S, device="cuda", generator=g)
    lab = torch.randint(0, 4, (B, 1, S, S), device="cuda", generator=g)
    return img, lab


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def b200seg_arm(block, B, S, steps, warmup):
    torch.manual_seed(0)
    net = b200seg.UNet2D(1, 4, 32, block=block).cuda()
    ema = b200seg.UNet2D(1, 4, 32, block=block).cuda()
    ema.load_state_dict(net.state_dict())
    opt = FusedAdamWEMA(net, ema, amp=True)
    crit = b200seg.DiceCELoss(weight=torch.tensor(CE_WEIGHT))
    img, lab = data(B, S)
    net.train()

    def step():
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss = crit(net(img), lab)
        opt.scale_loss(loss).backward()
        opt.step()
    return time_steps(step, steps, warmup)


def stock_arm(block, B, S, steps, warmup, benchmark, channels_last):
    torch.backends.cudnn.benchmark = benchmark
    torch.manual_seed(0)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    net = UNet2DRef(1, 4, 32, block=block).cuda().to(memory_format=fmt)
    ema = UNet2DRef(1, 4, 32, block=block).cuda().to(memory_format=fmt)
    ema.load_state_dict(net.state_dict())
    opt = torch.optim.AdamW(net.parameters(), lr=1e-3, eps=1e-5, weight_decay=0.05, fused=True)
    scaler = torch.amp.GradScaler("cuda")
    w = torch.tensor(CE_WEIGHT, device="cuda")
    img, lab = data(B, S)
    img = img.contiguous(memory_format=fmt)
    p_net, p_ema = list(net.parameters()), list(ema.parameters())
    b_net, b_ema = list(net.buffers()), list(ema.buffers())
    net.train()

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            out = net(img)
            loss = torch.nn.functional.cross_entropy(out, lab.squeeze(1), weight=w) + olosses.dice_loss(out, lab)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        with torch.no_grad():
            torch._foreach_lerp_(p_ema, p_net, 0.01)
            for eb, mb in zip(b_ema, b_net):
                eb.copy_(mb)
    ms = time_steps(step, steps, warmup)
    torch.backends.cudnn.benchmark = False
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", nargs="+", default=["SingleConv", "BasicBlock"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-stock", action="store_true", help="time the b200seg arm only")
    a = ap.parse_args()
    info = card()
    for block in a.blocks:
        res = {"workload": "acdc_2d_%s" % {"SingleConv": "unet", "BasicBlock": "resunet"}[block], "block": block,
               "batch": a.batch, "size": a.size, "amp": True, "steps": a.steps, "warmup": a.warmup, **info}
        ms = b200seg_arm(block, a.batch, a.size, a.steps, a.warmup)
        res["b200seg_ms_per_step"] = ms
        res["b200seg_images_per_s"] = a.batch * 1000.0 / ms
        if not a.no_stock:
            arms = {}
            for name, bm, cl in (("default", False, False), ("benchmark", True, False), ("benchmark_channels_last", True, True)):
                arms[name] = stock_arm(block, a.batch, a.size, a.steps, a.warmup, bm, cl)
            best = min(arms, key=arms.get)
            res["stock_ms_per_step"] = arms
            res["stock_best"] = best
            res["stock_best_images_per_s"] = a.batch * 1000.0 / arms[best]
            res["speedup_vs_stock_best"] = arms[best] / ms
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
