"""CPU: b200seg.SwinUNETR's state_dict contract and its module wiring with every C-ABI op emulated in PyTorch
(tests/emu_swin.py), against the reference-pinned oracle (oracle/swin_unetr.py) in fp64."""
import pytest
import torch

import b200seg
import emu_swin
from oracle import losses as olosses
from oracle import swin_unetr as osw
from oracle import unet3d as ounet
from oracle.synth import make_volume
from util import global_l2, load_golden, rel_err


def test_state_dict_contract():
    g = load_golden("swin_unetr_small")
    c = g["cfg"]
    net = b200seg.SwinUNETR(c["size"], c["in_ch"], c["classes"], feature_size=c["feature_size"])
    keys = [k for k in net.state_dict() if not k.endswith("relative_position_index")]
    assert keys == list(g["shapes"])
    assert all(tuple(net.state_dict()[k].shape) == tuple(g["shapes"][k]) for k in keys)
    with pytest.raises(ValueError):
        b200seg.SwinUNETR(c["size"], c["in_ch"], c["classes"], feature_size=20)          # feature_size % 12 (the reference's check)


@pytest.mark.parametrize("name", ["swin_block_a", "swin_block_b", "swin_block_c"])
@pytest.mark.parametrize("chunk", [64, 1])
def test_window_attention_core_reproduces_block_fixtures(name, chunk):
    """oracle.swin_ops.window_attention_core, the fp64 statement the GPU window-attention tests compare against, composed
    as LayerNorm -> qkv Linear -> window_attention_core -> proj reproduces the reference's SwinTransformerBlock
    .forward_part1 (padding, shift, clamped window) and every one of its gradients, including the bias table and qkv_b."""
    import torch.nn.functional as F
    from oracle import swin_ops as so
    g = load_golden(name)
    cfg = g["cfg"]
    p = {k: v.double().clone().requires_grad_(True) for k, v in g["params"].items()}
    x = g["x"].double().clone().requires_grad_(True)
    xn = F.layer_norm(x, (x.shape[-1],), p["norm1_w"], p["norm1_b"])
    qkv = F.linear(xn, p["qkv_w"], p["qkv_b"])
    att = so.window_attention_core(qkv, p["qkv_b"], p["bias_table"], cfg["heads"], cfg["window"], cfg["shift"], chunk=chunk)
    y = F.linear(att, p["proj_w"], p["proj_b"])
    y.backward(g["gy"].double())
    # the fixtures are the reference's fp32 numbers: 4e-7 is the largest distance measured
    assert rel_err(y, g["y"]) < 2e-6
    assert rel_err(x.grad, g["dx"]) < 2e-6
    errs = {k: rel_err(p[k].grad, g["dparams"][k]) for k in p}
    assert max(errs.values()) < 2e-6, errs


def test_orchestration_matches_oracle(monkeypatch):
    emu_swin.install(monkeypatch)
    size, classes, fs = (64, 32, 32), 3, 12          # deepest level 2x1x1: InstanceNorm needs more than one voxel
    shapes = osw.swin_unetr_param_shapes(1, classes, fs)
    sd = ounet.make_state_dict(shapes, seed=7)
    for k in sd:
        if k.endswith("norm1.weight") or k.endswith("norm2.weight") or k.endswith("norm.weight"):
            sd[k] = 1.0 + 0.1 * sd[k] / sd[k].abs().max()
        if k.endswith("relative_position_bias_table"):
            sd[k] = sd[k] * 3.0
    net = b200seg.SwinUNETR(size, 1, classes, feature_size=fs)
    missing = net.load_state_dict(sd, strict=False)
    assert all(k.endswith("relative_position_index") for k in missing.missing_keys) and not missing.unexpected_keys
    img, lab = make_volume(1, *size, classes, seed=8)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    logits = net(img)
    w = torch.tensor([0.5, 1.0, 2.0])
    b200seg.DiceCELoss(weight=w)(logits, lab).backward()
    s64 = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    l64 = osw.swin_unetr_forward(s64, img.double())
    olosses.total_loss(l64, lab, w.double()).backward()
    assert rel_err(logits, l64) < 2e-4
    ours = {k: p.grad for k, p in net.named_parameters()}
    assert all(v is not None for v in ours.values()), [k for k, v in ours.items() if v is None]
    g64 = {k: v.grad for k, v in s64.items()}
    assert set(ours) == set(g64)
    err = global_l2(ours, g64)
    print("swin emulated-orchestration grad L2 err vs fp64 oracle: %.2e" % err)
    assert err < 5e-2
