"""CPU: UNETR — the oracle against the reference fixture (oracle/make_golden_unetr.py), b200seg.UNETR's state_dict
contract and MONAI initialisation, get_model dispatch and the configurations the H100 path rejects, and the model's
wiring with every C-ABI op emulated in PyTorch (tests/emu_unetr.py) against the oracle in fp64."""
import types

import pytest
import torch

import b200seg
import emu_unetr
from oracle import losses as olosses
from oracle import make_golden_unetr as standin
from oracle import unetr as ounetr
from oracle.synth import make_volume
from util import global_l2, load_golden, rel_err


def _cfg():
    return load_golden("unetr_small")["cfg"]


def _net(c, **kw):
    return b200seg.UNETR(c["in_ch"], c["classes"], c["size"], feature_size=c["feature_size"], hidden_size=c["hidden"],
                         mlp_dim=c["mlp"], num_heads=c["heads"], **kw)


def test_oracle_matches_reference_fixture():
    g = load_golden("unetr_small")
    c = g["cfg"]
    sd = {k: v.requires_grad_(True) for k, v in ounetr.seeded_state_dict(g["shapes"], c["state_seed"]).items()}
    img, lab = make_volume(c["batch"], *c["size"], c["classes"], seed=c["data_seed"], in_ch=c["in_ch"])
    lo = ounetr.unetr_forward(sd, img, c["heads"])
    loss = olosses.total_loss(lo, lab, torch.tensor(c["ce_weight"]))
    loss.backward()
    ls = ounetr.voxel_sample(lo.detach(), g["stride"])
    assert rel_err(ls, g["logits"].float()) < 2e-3          # the fixture stores fp16 logits of every 15th voxel
    assert (ls.argmax(1).to(torch.uint8) == g["argmax"]).float().mean().item() > 0.999
    assert abs(loss.item() - g["loss"]) < 1e-5
    for k, d in g["grad_digest"].items():
        gk = sd[k].grad.double()
        assert abs(gk.abs().sum().item() - d["abs"]) <= 1e-4 * d["abs"] + 1e-12, k
        assert abs((gk * gk).sum().item() - d["sq"]) <= 1e-4 * d["sq"] + 1e-24, k


def test_state_dict_contract():
    g = load_golden("unetr_small")
    c = g["cfg"]
    net = _net(c)
    assert list(net.state_dict()) == list(g["shapes"])
    assert all(tuple(v.shape) == tuple(g["shapes"][k]) for k, v in net.state_dict().items())
    sd = ounetr.seeded_state_dict(g["shapes"], c["state_seed"])
    net.load_state_dict(sd)                                  # a state_dict keyed like the reference's loads as is
    vit = standin.ViT(c["in_ch"], c["size"], (16, 16, 16), hidden_size=c["hidden"], mlp_dim=c["mlp"], num_layers=12,
                      num_heads=c["heads"], pos_embed="perceptron")
    vit.load_state_dict(net.vit.state_dict())                # and ours loads back into the MONAI-semantics stand-in
    assert all(torch.equal(v, sd["vit." + k]) for k, v in vit.state_dict().items())


def test_init_matches_monai():
    """Same seed, same draws: the ViT (trunc_normal(0.02) position table and patch Linear, zero bias, default-initialised
    transformer Linears) and the transposed-conv chain initialise exactly as the MONAI-semantics stand-ins."""
    c = _cfg()
    args = (c["in_ch"], c["size"], (16, 16, 16))
    kw = dict(hidden_size=c["hidden"], mlp_dim=c["mlp"], num_layers=12, num_heads=c["heads"], pos_embed="perceptron")
    from b200seg import unetr as ur
    torch.manual_seed(5)
    ours = ur.ViT(*args, **kw).state_dict()
    torch.manual_seed(5)
    ref = standin.ViT(*args, **kw).state_dict()
    assert list(ours) == list(ref)
    assert all(torch.equal(ours[k], ref[k]) for k in ref)
    pe = ours["patch_embedding.position_embeddings"]
    assert pe.abs().max() <= 2.0 and 0.01 < pe.std().item() < 0.03
    assert not ours["patch_embedding.patch_embeddings.1.bias"].any()
    pr = dict(spatial_dims=3, in_channels=c["hidden"], out_channels=32, num_layer=2, kernel_size=3, stride=1,
              upsample_kernel_size=2, norm_name="instance")
    torch.manual_seed(6)
    a = ur.UnetrPrUpBlock(**pr).state_dict()
    torch.manual_seed(6)
    b = standin.UnetrPrUpBlock(**pr).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in b)


def _args(**kw):
    a = dict(dimension="3d", model="unetr", in_chan=1, classes=14, training_size=[96, 96, 96])
    a.update(kw)
    return types.SimpleNamespace(**a)


def test_get_model_builds_the_reference_config():
    net = b200seg.get_model(_args())
    assert isinstance(net, b200seg.UNETR)
    assert net.feat_size == (6, 6, 6) and net.hidden_size == 768
    shapes = ounetr.unetr_param_shapes(1, 14, (96, 96, 96))
    assert list(net.state_dict()) == list(shapes)
    assert all(tuple(v.shape) == shapes[k] for k, v in net.state_dict().items())
    assert isinstance(b200seg.get_model(_args(training_size=[16, 192, 192], classes=4), pretrain=True), b200seg.UNETR)


def test_rejections():
    c = _cfg()
    with pytest.raises(ValueError):
        _net(c, pos_embed="conv")
    with pytest.raises(KeyError):
        _net(c, pos_embed="learned")
    with pytest.raises(ValueError):
        _net(c, conv_block=True)
    with pytest.raises(ValueError):
        _net(c, dropout_rate=0.1)
    with pytest.raises(AssertionError):
        _net(c, dropout_rate=1.5)
    with pytest.raises(ValueError):
        _net(c, norm_name="batch")
    with pytest.raises(ValueError):
        _net(c, res_block=False)
    with pytest.raises(ValueError):
        b200seg.UNETR(1, 3, (32, 40, 64), hidden_size=128, mlp_dim=256, num_heads=2)     # 40 % 16
    with pytest.raises(AssertionError):
        b200seg.UNETR(1, 3, (32, 48, 64), hidden_size=130, mlp_dim=256, num_heads=4)     # hidden % heads
    with pytest.raises(ValueError):
        b200seg.UNETR(1, 3, (32, 48, 64), hidden_size=128, mlp_dim=256, num_heads=4)     # head size 32
    net = _net(c)
    with pytest.raises(b200seg.B200SegError):
        net(torch.zeros(1, 1, *c["size"]))                   # CPU tensors: no fallback


def test_orchestration_matches_oracle(monkeypatch):
    emu_unetr.install(monkeypatch)
    size, classes, heads, hidden = (32, 32, 48), 3, 2, 128
    shapes = ounetr.unetr_param_shapes(1, classes, size, 16, hidden, 256)
    sd = ounetr.seeded_state_dict(shapes, 9)
    net = b200seg.UNETR(1, classes, size, feature_size=16, hidden_size=hidden, mlp_dim=256, num_heads=heads)
    net.load_state_dict(sd)
    img, lab = make_volume(2, *size, classes, seed=10)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    logits = net(img)
    w = torch.tensor([0.5, 1.0, 2.0])
    b200seg.DiceCELoss(weight=w)(logits, lab).backward()
    s64 = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    l64 = ounetr.unetr_forward(s64, img.double(), heads)
    olosses.total_loss(l64, lab, w.double()).backward()
    assert rel_err(logits, l64) < 2e-4
    ours = {k: p.grad for k, p in net.named_parameters()}
    assert all(v is not None for v in ours.values()), [k for k, v in ours.items() if v is None]
    g64 = {k: v.grad for k, v in s64.items()}
    assert set(ours) == set(g64)
    err = global_l2(ours, g64)
    worst = max(rel_err(ours[k], g64[k]) for k in g64 if k.startswith("vit."))
    print("unetr emulated-orchestration grad L2 err vs fp64 oracle: %.2e (worst ViT tensor %.2e)" % (err, worst))
    assert err < 1e-4
    assert rel_err(ours["vit.patch_embedding.position_embeddings"], g64["vit.patch_embedding.position_embeddings"]) < 1e-3
