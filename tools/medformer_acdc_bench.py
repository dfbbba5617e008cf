#!/usr/bin/env python
"""medformer_acdc_bench.py — training-step time of the ACDC MedFormer (config/acdc/medformer_3d.yaml: map 2x6x6, 4 heads
per level, fusion 256 / 4 heads, aux loss) at the reference README's crop and batch (3 x 1 x 16 x 192 x 192, 4 classes)
on one GPU, for b200seg and for the unmodified reference.

  python tools/medformer_acdc_bench.py [--rounds 3] [--steps 10] [--warmup 3] [--out DIR]
  python tools/medformer_acdc_bench.py --profile [--out DIR]

One step = zero_grad -> autocast fp16 forward -> 0.5 * (CE(weight [0.5,1,1,1]) + Dice) on each of the two outputs ->
scaled backward -> AdamW(eps 1e-5, wd 0.05) -> EMA (training/utils.py, train_ddp.py:171-215).
  b200seg   : b200seg.get_model with b200seg.DiceCELoss and b200seg.train.FusedAdamWEMA.
  reference : the reference's own MedFormer and DiceLoss from oracle/_ref (as bench.py --impl reference loads them),
              under stock torch autocast + GradScaler + torch.optim.AdamW and a foreach EMA, cuDNN default.
The arms alternate for --rounds rounds (CUDA events over --steps steps after --warmup each) and the median per arm is
reported with the card's name, power limit and SM clock read in the same run.  --profile records one b200seg step with
torch.profiler (CUDA activities) and writes the kernel table plus the share of the step's kernel time spent in the
B-MHA (biattn), map-generation and token-attention (mhsa) kernels under --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                   # noqa: E402

import b200seg                                 # noqa: E402
from b200seg.train import FusedAdamWEMA        # noqa: E402

ACDC = dict(map_size=[2, 6, 6], conv_num=[2, 0, 0, 0, 0, 0, 2, 2], trans_num=[0, 2, 2, 2, 2, 2, 0, 0],
            num_heads=[1, 4, 4, 4, 4, 4, 1, 1], fusion_depth=2, fusion_dim=256, fusion_heads=4,
            kernel_size=[[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
            scale=[[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2]], aux_loss=True)
CE_WEIGHT = [0.5, 1.0, 1.0, 1.0]
AUX_WEIGHT = [0.5, 0.5]
CLASSES = 4


def card():
    if not torch.cuda.is_available():
        raise SystemExit("medformer_acdc_bench.py measures on a CUDA device; none is visible")
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        p, c, cm = (float(v) for v in q.stdout.strip().splitlines()[0].split(","))
        info.update(power_limit_w=p, sm_clock_mhz=c, sm_clock_max_mhz=cm)
    except Exception as e:      # noqa
        info["nvidia_smi"] = "unavailable: %r" % (e,)
    return info


def args_ns():
    c = dict(ACDC)
    return types.SimpleNamespace(dimension="3d", model="medformer", in_chan=1, classes=CLASSES, base_chan=32,
                                 conv_block="BasicBlock", expansion=4, attn_drop=0.0, proj_drop=0.0,
                                 proj_type="depthwise", norm="in", act="relu", down_scale=c.pop("scale"), **c)


def data(B, D, H, W):
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randn(B, 1, D, H, W, device="cuda", generator=g)
    lab = torch.randint(0, CLASSES, (B, 1, D, H, W), device="cuda", generator=g)
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


def b200seg_step(img, lab):
    torch.manual_seed(0)
    net = b200seg.get_model(args_ns()).cuda()
    ema = b200seg.get_model(args_ns()).cuda()
    ema.load_state_dict(net.state_dict())
    opt = FusedAdamWEMA(net, ema, amp=True)
    crit = b200seg.DiceCELoss(weight=torch.tensor(CE_WEIGHT))
    net.train()

    def step():
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            res = net(img)
            loss = sum(w * crit(r, lab) for w, r in zip(AUX_WEIGHT, res))
        opt.scale_loss(loss).backward()
        opt.step()
    return step


def reference_step(img, lab):
    import bench
    ref = bench.reference_classes()
    if ref is None:
        raise SystemExit("the reference MedFormer is not importable from oracle/_ref: run `python __graft_entry__.py "
                         "build` where the reference sources are available")
    kw = dict(ACDC)
    torch.manual_seed(0)

    def make():
        return ref["MedFormer"](1, CLASSES, 32, conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0,
                                proj_type="depthwise", norm="in", act="relu", **kw).cuda()
    net, ema = make(), make()
    ema.load_state_dict(net.state_dict())
    opt = torch.optim.AdamW(net.parameters(), lr=1e-3, eps=1e-5, weight_decay=0.05)
    scaler = torch.amp.GradScaler("cuda")
    ce = torch.nn.CrossEntropyLoss(weight=torch.tensor(CE_WEIGHT, device="cuda"))
    dl = ref["DiceLoss"]()
    p_net, p_ema = list(net.parameters()), list(ema.parameters())
    net.train()

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            res = net(img)
            loss = sum(w * (ce(r, lab.squeeze(1)) + dl(r, lab)) for w, r in zip(AUX_WEIGHT, res))
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        with torch.no_grad():
            torch._foreach_lerp_(p_ema, p_net, 0.01)
    return step


ATTN = ("biattn", "mapgen", "mhsa")


def profile(img, lab, out):
    from torch.profiler import ProfilerActivity, profile as tprofile
    step = b200seg_step(img, lab)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t and e.device_type == torch.autograd.DeviceType.CUDA:
            rows[e.key] = rows.get(e.key, 0.0) + t
    total = sum(rows.values())
    share = {a: sum(t for k, t in rows.items() if a in k) / total for a in ATTN}
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "medformer_acdc_profile.txt"), "w") as f:
        f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=60))
    return {"table": os.path.join(out, "medformer_acdc_profile.txt"), "kernel_time_ms": total / 1000.0, "share": share,
            "attention_share": sum(share.values()),
            "top": sorted(((k, t / 1000.0) for k, t in rows.items()), key=lambda kv: -kv[1])[:15]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=3)
    ap.add_argument("--crop", type=int, nargs=3, default=[16, 192, 192])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "medformer_acdc_bench"),
                    help="directory for the --profile table (default: a directory under the system temp dir)")
    a = ap.parse_args()
    if a.rounds < 3 and not a.profile:
        raise SystemExit("--rounds must be at least 3")
    res = {"workload": "medformer_acdc", "batch": a.batch, "crop": a.crop, "classes": CLASSES, "amp": True, **card()}
    img, lab = data(a.batch, *a.crop)
    if a.profile:
        res["profile"] = profile(img, lab, a.out)
    else:
        arms = {"b200seg": b200seg_step(img, lab), "reference": reference_step(img, lab)}
        times = {k: [] for k in arms}
        for _ in range(a.rounds):
            for name, step in arms.items():
                times[name].append(time_steps(step, a.steps, a.warmup))
        res.update(steps=a.steps, warmup=a.warmup, rounds=a.rounds, ms_per_step=times,
                   median_ms={k: statistics.median(v) for k, v in times.items()})
        res["speedup_vs_reference"] = res["median_ms"]["reference"] / res["median_ms"]["b200seg"]
        res.update({"after_" + k: v for k, v in card().items() if k.startswith("sm_clock")})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
