"""CPU: the 2D UNet / ResUNet (model/dim2/unet.py) — state_dict contract, factory dispatch, and a training step with
the C-ABI ops emulated in PyTorch (tests/emu_bn.py) against fixtures made by the unmodified reference class."""
import types

import pytest
import torch

import b200seg
from oracle.make_golden_unet2d import batch, seeded_state_dict
from util import load_golden, rel_err
import emu_bn


def _args(**kw):
    a = types.SimpleNamespace(dimension="2d", model="unet", in_chan=1, base_chan=32, classes=4, block="SingleConv")
    a.__dict__.update(kw)
    return a


# numbers of the unmodified reference class at base 32, 4 classes
@pytest.mark.parametrize("model,block,params,tensors,entries,bns", [
    ("resunet", "BasicBlock", 18225220, 137, 263, 42),
    ("unet", "SingleConv", 7240260, 62, 113, 17),
])
def test_state_dict_contract(model, block, params, tensors, entries, bns):
    net = b200seg.get_model(_args(model=model, block=block))
    assert isinstance(net, b200seg.UNet2D)
    ps = list(net.parameters())
    assert sum(p.numel() for p in ps) == params
    assert len(ps) == tensors
    sd = net.state_dict()
    assert len(sd) == entries
    assert sum(isinstance(m, torch.nn.BatchNorm2d) for m in net.modules()) == bns
    assert sum(k.endswith("num_batches_tracked") for k in sd) == bns
    # strict loading both ways, and the holders draw the same initialisation under the same seed
    torch.manual_seed(3)
    a = b200seg.get_model(_args(model=model, block=block))
    torch.manual_seed(3)
    b = b200seg.get_model(_args(model=model, block=block))
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    a.load_state_dict(net.state_dict(), strict=True)
    net.load_state_dict(a.state_dict(), strict=True)


@pytest.mark.parametrize("name", ["unet2d_single", "unet2d_basic"])
def test_keys_and_shapes_match_reference(name):
    g = load_golden(name)
    cfg = g["cfg"]
    net = b200seg.UNet2D(1, cfg["classes"], cfg["base"], block=cfg["block"])
    sd = net.state_dict()
    assert list(sd) == g["keys"]
    assert {k: tuple(v.shape) for k, v in sd.items()} == g["shapes"]
    assert sd[[k for k in sd if k.endswith("num_batches_tracked")][0]].dtype == torch.int64


def test_factory_2d_dispatch_and_errors():
    assert isinstance(b200seg.get_model(_args(model="unet")), b200seg.UNet2D)
    assert isinstance(b200seg.get_model(_args(model="resunet", block="BasicBlock")), b200seg.UNet2D)
    with pytest.raises(ValueError):
        b200seg.get_model(_args(model="unet"), pretrain=True)
    for m in ("unet++", "attention_unet", "daunet", "medformer", "transunet", "swinunet"):
        with pytest.raises(ValueError):
            b200seg.get_model(_args(model=m))
    with pytest.raises(ValueError):
        b200seg.get_model(_args(model="unet", block="Bottleneck"))
    with pytest.raises(ValueError):
        b200seg.get_model(types.SimpleNamespace(dimension="3d", model="unet", in_chan=1, base_chan=8, classes=4,
                                                down_scale=[[2, 2, 2]] * 4, norm="bn", kernel_size=[[3, 3, 3]] * 5,
                                                block="BasicBlock"))


def test_holder_settings_that_the_kernels_do_not_implement_raise(monkeypatch):
    emu_bn.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    img, _ = batch(2, 32, 32, 4, 0)
    for attr, val in (("momentum", None), ("affine", False), ("track_running_stats", False)):
        net = b200seg.UNet2D(1, 4, 8, block="SingleConv")
        setattr(net.inc.conv2.conv.norm, attr, val)
        with pytest.raises(ValueError):
            net(img)
    net = b200seg.UNet2D(1, 4, 8, block="BasicBlock")
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        net(torch.randn(1, 1, 16, 16))          # down4 sees 1x1 per channel at batch 1


def _run_steps(net, cfg, dev="cpu"):
    """Three training forwards (CE + Dice, backward, no parameter update) on the fixture's batches, as
    oracle/make_golden_unet2d.py runs the reference; batches go to `dev`, results come back to the CPU."""
    B, H, W = cfg["shape"]
    w = torch.tensor(cfg["ce_weight"])
    out = {}
    for step, seed in enumerate(cfg["data_seeds"]):
        img, lab = (t.to(dev) for t in batch(B, H, W, cfg["classes"], seed))
        net.train()
        net.zero_grad(set_to_none=True)
        logits = net(img)
        loss = b200seg.DiceCELoss(weight=w)(logits, lab)
        loss.backward()
        if step == 0:
            out.update(logits=logits.detach().float().cpu(), loss=loss.item(),
                       grads={k: p.grad.to("cpu", copy=True) for k, p in net.named_parameters()},
                       running_1={k: v.to("cpu", copy=True) for k, v in net.state_dict().items() if "running_" in k or "num_batches" in k})
            net.eval()
            with torch.no_grad():
                out["eval_1"] = net(img).float().cpu()
    out["running_3"] = {k: v.to("cpu", copy=True) for k, v in net.state_dict().items() if "running_" in k or "num_batches" in k}
    net.eval()
    with torch.no_grad():
        out["eval_3"] = net(batch(B, H, W, cfg["classes"], cfg["data_seeds"][0])[0].to(dev)).float().cpu()
    return out


@pytest.mark.parametrize("name", ["unet2d_single", "unet2d_basic"])
def test_orchestration_matches_reference(monkeypatch, name):
    emu_bn.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    g = load_golden(name)
    cfg = g["cfg"]
    net = b200seg.UNet2D(1, cfg["classes"], cfg["base"], block=cfg["block"])
    net.load_state_dict(seeded_state_dict(net, cfg["state_seed"]))
    r = _run_steps(net, cfg)
    assert rel_err(r["logits"], g["logits"]) < 1e-4
    assert abs(r["loss"] - g["loss"]) < 1e-4
    for k, d in g["grad_digest"].items():
        gk = r["grads"][k].double()
        assert abs(gk.sum().item() - d["sum"]) <= 1e-3 * d["abs"] + 1e-6, k
        assert abs((gk * gk).sum().item() - d["sq"]) <= 1e-3 * d["sq"] + 1e-9, k
    for k, v in g["grad_small"].items():
        # conv_ch.bias of a ResUNet feeds only BatchNorms, so its true gradient is 0 and both sides hold round-off
        assert (r["grads"][k] - v).abs().max() <= 1e-3 * v.abs().max() + 1e-7, k
    for key in ("running_1", "running_3"):
        for k, v in g[key].items():
            if v.dtype == torch.int64:
                assert torch.equal(r[key][k], v), k
            else:
                assert torch.allclose(r[key][k], v, rtol=1e-4, atol=1e-5), k
    assert rel_err(r["eval_1"], g["eval_logits_1"].float()) < 2e-3          # fixture stored in fp16
    assert rel_err(r["eval_3"], g["eval_logits_3"].float()) < 2e-3
