"""Write tests/golden/unet2d_{single,basic}.pt from the UNMODIFIED reference 2D UNet (model/dim2/unet.py).

Runs only where the reference checkout exists (B200SEG_REFERENCE, default /root/reference).  model/dim2/conv_layers.py
imports timm for its ConvNeXt / MBConv blocks, and timm is not installed: a stub module providing the two names it
imports is registered for this script only (neither the SingleConv nor the BasicBlock path uses them).

Per block, on CPU in fp32, with a seeded state_dict (weights, BatchNorm affine parameters and running statistics all
drawn from the seed so that no parameter sits at its default):
  * step 1: train-mode forward on batch 0, CE(weight) + Dice, backward -> logits, loss, gradient digests, and the
    running statistics after the step;
  * eval-mode logits on batch 0 after step 1;
  * steps 2 and 3: train-mode forward/backward on batches 1 and 2 (no parameter update) -> running statistics and
    eval-mode logits after three steps;
  * the state_dict key list and shapes (the state_dict itself is regenerated from its seed by seeded_state_dict).
Eval-mode logits are stored in fp16 to keep the fixtures small.
Usage:  python oracle/make_golden_unet2d.py
"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("B200SEG_REFERENCE", "/root/reference")

CASES = {
    # name: (block, base, classes, B, H, W, ce_weight)
    "unet2d_single": ("SingleConv", 8, 4, 4, 48, 48, [0.5, 1.0, 1.0, 2.0]),
    "unet2d_basic": ("BasicBlock", 8, 4, 4, 48, 48, [0.5, 1.0, 1.0, 2.0]),
}


def import_reference():
    sys.path.insert(0, REF)
    timm = types.ModuleType("timm")
    timm_models = types.ModuleType("timm.models")
    timm_layers = types.ModuleType("timm.models.layers")
    timm_layers.trunc_normal_ = torch.nn.init.trunc_normal_
    timm_layers.DropPath = torch.nn.Identity
    timm.models, timm_models.layers = timm_models, timm_layers
    sys.modules.update({"timm": timm, "timm.models": timm_models, "timm.models.layers": timm_layers})
    for pkg, sub in (("model", "model"), ("model.dim2", "model/dim2")):
        m = types.ModuleType(pkg)
        m.__path__ = [os.path.join(REF, sub)]
        sys.modules[pkg] = m
    from model.dim2.unet import UNet          # noqa
    from training.losses import DiceLoss      # noqa
    return UNet, DiceLoss


def seeded_state_dict(ref, seed):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in ref.state_dict().items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(int(torch.randint(0, 50, (1,), generator=g)), dtype=torch.long)
        elif k.endswith("running_var"):
            sd[k] = torch.rand(v.shape, generator=g) * 1.5 + 0.25
        elif k.endswith("running_mean"):
            sd[k] = torch.randn(v.shape, generator=g) * 0.3
        elif ".norm.weight" in k:
            # gamma of both signs and some exactly zero: the fold must not divide by it
            w = torch.randn(v.shape, generator=g) * 0.5 + 0.8
            w[::7] = -w[::7].abs()
            w[3::11] = 0.0
            sd[k] = w
        elif ".norm.bias" in k:
            sd[k] = torch.randn(v.shape, generator=g) * 0.2
        else:
            fan_in = v[0].numel() if v.dim() > 1 else 1
            sd[k] = torch.randn(v.shape, generator=g) * (2.0 / fan_in) ** 0.5 if v.dim() > 1 else torch.randn(v.shape, generator=g) * 0.1
    return sd


def batch(B, H, W, classes, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(B, 1, H, W, generator=g)
    img = img + torch.nn.functional.avg_pool2d(torch.randn(B, 1, H, W, generator=g) * 4, 9, 1, 4)
    lab = torch.randint(0, classes, (B, 1, H // 8, W // 8), generator=g)
    lab = torch.nn.functional.interpolate(lab.float(), size=(H, W), mode="nearest").long()
    return img, lab


def digest(t):
    t = t.detach().double().flatten()
    idx = torch.linspace(0, t.numel() - 1, min(t.numel(), 64)).long()
    return {"sum": t.sum().item(), "abs": t.abs().sum().item(), "sq": (t * t).sum().item(), "sample": t[idx].float()}


def running(ref):
    return {k: v.clone() for k, v in ref.state_dict().items() if "running_" in k or "num_batches" in k}


def main():
    torch.set_num_threads(8)
    UNet, DiceLoss = import_reference()
    for name, (block, base, classes, B, H, W, w) in CASES.items():
        torch.manual_seed(0)
        ref = UNet(1, classes, base, block=block)
        sd = seeded_state_dict(ref, seed=11)
        ref.load_state_dict(sd)
        weight = torch.tensor(w)
        out = {"cfg": {"block": block, "base": base, "classes": classes, "shape": (B, H, W), "ce_weight": w,
                       "state_seed": 11, "data_seeds": [100, 101, 102]},
               "keys": list(sd), "shapes": {k: tuple(v.shape) for k, v in sd.items()}}
        for step, seed in enumerate([100, 101, 102]):
            img, lab = batch(B, H, W, classes, seed)
            ref.train()
            ref.zero_grad(set_to_none=True)
            logits = ref(img)
            loss = torch.nn.CrossEntropyLoss(weight=weight)(logits, lab.squeeze(1)) + DiceLoss()(logits, lab)
            loss.backward()
            if step == 0:
                out["logits"] = logits.detach().clone()
                out["loss"] = loss.item()
                out["grad_digest"] = {k: digest(p.grad) for k, p in ref.named_parameters()}
                out["grad_small"] = {k: p.grad.clone() for k, p in ref.named_parameters() if p.numel() <= 4096}
                out["running_1"] = running(ref)
                ref.eval()
                with torch.no_grad():
                    out["eval_logits_1"] = ref(img).half()
        out["running_3"] = running(ref)
        img0, _ = batch(B, H, W, classes, 100)
        ref.eval()
        with torch.no_grad():
            out["eval_logits_3"] = ref(img0).half()
        # the stock-torch restatement (oracle/unet2d.py) must reproduce the reference class
        sys.path.insert(0, ROOT)
        from oracle.unet2d import UNet2DRef
        ora = UNet2DRef(1, classes, base, block=block)
        assert list(ora.state_dict()) == out["keys"], "oracle key order != reference registration order"
        ora.load_state_dict(sd)
        ora.train()
        img, _ = batch(B, H, W, classes, 100)
        err = ((ora(img) - out["logits"]).abs().max() / out["logits"].abs().max()).item()
        print("%-14s oracle-vs-reference logits %.2e" % (name, err))
        assert err < 1e-5, "oracle restatement diverges from the reference"
        path = os.path.join(ROOT, "tests", "golden", name + ".pt")
        torch.save(out, path)
        print("%-14s loss %.6f  -> %s (%d bytes)" % (name, out["loss"], path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
