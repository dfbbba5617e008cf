"""GPU: the BatchNorm kernels and the per-channel mode of the convolutions against fp64, and the 2D UNet / ResUNet
against fixtures made by the unmodified reference class (model/dim2/unet.py)."""
import pytest
import torch
import torch.nn.functional as F

import b200seg
from b200seg import _lib
from b200seg import batchnorm as bn
from b200seg.ops import PackedWeights, instnorm_stats
from b200seg.train import FusedAdamWEMA
from oracle.make_golden_unet2d import seeded_state_dict
from test_unet2d_host import _run_steps
from util import load_golden, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _holder(C, seed, training=True):
    g = torch.Generator().manual_seed(seed)
    h = torch.nn.BatchNorm2d(C, momentum=0.1 + 0.05 * (seed % 3)).to(DEV)
    with torch.no_grad():
        w = torch.randn(C, generator=g) * 0.7
        w[::5] = 0.0
        w[1::5] = -w[1::5].abs() - 0.1
        h.weight.copy_(w)
        h.bias.copy_(torch.randn(C, generator=g) * 0.3)
        h.running_mean.copy_(torch.randn(C, generator=g) * 0.2)
        h.running_var.copy_(torch.rand(C, generator=g) + 0.5)
        h.num_batches_tracked.fill_(seed)
    h.train(training)
    return h


def _x(B, H, W, C, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1, H, W, C, generator=g) * (torch.rand(C, generator=g) * 2 + 0.1) + torch.randn(C, generator=g) * 3
    return x.to(DEV, dtype).contiguous()


@pytest.mark.parametrize("B,H,W,C", [(2, 1, 1, 8), (1, 1, 2, 16), (3, 5, 7, 32), (32, 16, 16, 64), (4, 8, 8, 1024)])
@pytest.mark.parametrize("training", [True, False])
def test_fwd_fold_against_fp64(B, H, W, C, training):
    x = _x(B, H, W, C, torch.float32, B * C + H)
    h = _holder(C, 3, training)
    ref = _holder(C, 3, training).double()
    sums = instnorm_stats(x, 0, C)
    table, mr = bn.bn_fold(h, sums, B * H * W)
    xr = x.double().permute(0, 4, 1, 2, 3).squeeze(2)
    ref(xr)
    for name in ("running_mean", "running_var"):
        assert rel_err(getattr(h, name), getattr(ref, name)) < 1e-6, name
    assert int(h.num_batches_tracked) == int(ref.num_batches_tracked)
    if training:
        # the fold's input is the sums; their own rounding (fp32 partials of x and x^2) is the sum kernel's business
        tot = sums.double().sum(0)
        mean = tot[:, 0] / (B * H * W)
        var = (tot[:, 1] / (B * H * W) - mean * mean).clamp_min(0)
        assert rel_err(mean, xr.mean((0, 2, 3))) < 1e-5
    else:
        mean, var = ref.running_mean, ref.running_var
    rstd = 1.0 / torch.sqrt(var + h.eps)
    s = h.weight.double() * rstd
    assert rel_err(table[:, 0], s) < 1e-6
    assert (table[:, 1].double() - (h.bias.double() - mean * s)).abs().max() < 1e-5 * (1 + mean.abs().max() * s.abs().max())
    assert rel_err(mr[:, 1], rstd) < 1e-6


def test_fold_rejects_one_value_per_channel():
    h = _holder(8, 1)
    with pytest.raises(ValueError, match="more than 1 value"):
        bn.bn_fold(h, torch.zeros(1, 8, 2, dtype=torch.float64, device=DEV), 1)
    with pytest.raises(_lib.B200SegError):
        _lib.call("b200seg_batchnorm_fwd_fold", torch.zeros(16, dtype=torch.float64, device=DEV).data_ptr(), 1, 8, 1.0,
                  h.weight.data_ptr(), h.bias.data_ptr(), h.running_mean.data_ptr(), h.running_var.data_ptr(), None,
                  0.1, 1e-5, 1, torch.empty(16, device=DEV).data_ptr(), torch.empty(16, device=DEV).data_ptr(), None)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("B,H,W,C", [(2, 3, 5, 8), (32, 8, 8, 128), (3, 4, 4, 1024)])
def test_apply_and_backward_against_fp64(dtype, B, H, W, C):
    tol = 1e-5 if dtype == torch.float32 else 2e-3
    x = _x(B, H, W, C, dtype, 7)
    h = _holder(C, 5)
    table, mr = bn.bn_fold(h, instnorm_stats(x, 0, C), B * H * W)
    y = bn.bn_apply(x, table, _lib.ACT_RELU)
    z = x.double() * table[:, 0].double() + table[:, 1].double()
    assert rel_err(y, F.relu(z)) < tol
    g = _x(B, H, W, C, dtype, 8) * 0.1
    # fp64 BatchNorm + ReLU backward through autograd, batch statistics as the kernels computed them
    xr = x.double().requires_grad_(True)
    gamma = h.weight.detach().double().requires_grad_(True)
    beta = h.bias.detach().double().requires_grad_(True)
    mean, var = xr.mean((0, 1, 2, 3)), xr.var((0, 1, 2, 3), unbiased=False)
    out = F.relu((xr - mean) / torch.sqrt(var + h.eps) * gamma + beta)
    out.backward(g.double())
    sums = bn.bn_bwd_reduce(g, x, table, _lib.ACT_RELU, mr)
    dg, db, coef = bn.bn_bwd_fold(sums, B * H * W, h.weight, mr, True)
    assert rel_err(dg, gamma.grad) < 10 * tol and rel_err(db, beta.grad) < 10 * tol
    dx = bn.bn_bwd_apply(g, x, table, _lib.ACT_RELU, coef)
    assert rel_err(dx, xr.grad) < 20 * tol
    # accumulation into another gradient, in place
    acc = _x(B, H, W, C, dtype, 9)
    want = acc.double() + xr.grad
    bn.bn_bwd_apply(g, x, table, _lib.ACT_RELU, coef, add=acc, out=acc)
    assert rel_err(acc, want) < 20 * tol
    # eval mode: the statistics are constants
    _, _, coef_e = bn.bn_bwd_fold(sums, B * H * W, h.weight, mr, False)
    dx_e = bn.bn_bwd_apply(g, x, table, _lib.ACT_RELU, coef_e)
    want_e = g.double() * (z > 0) * table[:, 0].double()
    assert rel_err(dx_e, want_e) < tol * 10


def _conv_ref(x, table, act, w, residual=None):
    a = x.double()
    if table is not None:
        a = a * table[:, 0].double() + table[:, 1].double()
    if act:
        a = F.relu(a)
    a = a.to(x.dtype).double().squeeze(1).permute(0, 3, 1, 2)
    y = F.conv2d(a, w.double(), padding=w.shape[-1] // 2).permute(0, 2, 3, 1).unsqueeze(1)
    if residual is not None:
        y = y.to(x.dtype).double() + residual.double()
    return y


@pytest.mark.parametrize("B,Cin,Cout,H", [(1, 64, 64, 32), (32, 128, 256, 16), (32, 512, 512, 16), (32, 1024, 512, 16),
                                          (64, 256, 256, 8), (32, 32, 32, 32)])
@pytest.mark.parametrize("transform", [True, False])
def test_per_channel_conv_against_fp64(B, Cin, Cout, H, transform):
    """fp16 tensor-core forward (with residual and output sums), data gradient and weight gradient in per-channel mode
    at batch sizes where the per-(sample, channel) tables of the InstanceNorm mode do not fit."""
    assert b200seg.ops.conv_algo(Cin, Cout, (1, 3, 3), torch.float16, 1) == _lib.ALGO_TC
    assert b200seg.ops.conv_algo(Cout, Cin, (1, 3, 3), torch.float16, 1) == _lib.ALGO_TC
    x = _x(B, H, H, Cin, torch.float16, Cin + B)
    g = torch.Generator().manual_seed(Cout)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (2.0 / (9 * Cin)) ** 0.5).to(DEV)
    w5 = w.view(Cout, Cin, 1, 3, 3)
    packs = PackedWeights().get([w5], torch.float16, 1)
    table = None
    act = _lib.ACT_NONE
    if transform:
        h = _holder(Cin, 2)
        table, _ = bn.bn_fold(h, instnorm_stats(x, 0, Cin), B * H * H)
        act = _lib.ACT_RELU
    res = _x(B, H, H, Cout, torch.float16, 3) if Cin != Cout else None
    y, ysum = bn.conv_pc_fwd(x, Cin, table, act, packs[0], Cout, (1, 3, 3), residual=res)
    yr = _conv_ref(x, table, act, w, res)
    assert rel_err(y, yr) < 5e-3
    yd = y.double()
    assert rel_err(ysum[..., 0], yd.sum((1, 2, 3))) < 1e-3
    dy = _x(B, H, H, Cout, torch.float16, 4) * 0.05
    dx, _ = bn.conv_pc_fwd(dy, Cout, None, _lib.ACT_NONE, packs[1], Cin, (1, 3, 3), want_stats=False)
    dxr = F.conv_transpose2d(dy.double().squeeze(1).permute(0, 3, 1, 2), w.double(), padding=1).permute(0, 2, 3, 1).unsqueeze(1)
    assert rel_err(dx, dxr) < 5e-3
    dw, _ = bn.conv_pc_wgrad(x, Cin, table, act, dy, Cout, (1, 3, 3), algo=_lib.ALGO_TC)      # no other path may run
    a = x.double()
    if table is not None:
        a = F.relu(a * table[:, 0].double() + table[:, 1].double())
    a = a.half().double().squeeze(1).permute(0, 3, 1, 2)
    wr = torch.zeros(Cout, Cin, 3, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    F.conv2d(a, wr, padding=1).backward(dy.double().squeeze(1).permute(0, 3, 1, 2))
    assert rel_err(dw.view(Cout, Cin, 3, 3), wr.grad) < 5e-3


@pytest.mark.parametrize("name", ["unet2d_single", "unet2d_basic"])
def test_model_fp32_matches_reference(name):
    g = load_golden(name)
    cfg = g["cfg"]
    net = b200seg.UNet2D(1, cfg["classes"], cfg["base"], block=cfg["block"])
    net.load_state_dict(seeded_state_dict(net, cfg["state_seed"]))
    net = net.to(DEV)
    r = _run_steps(net, cfg, DEV)
    assert rel_err(r["logits"], g["logits"]) < 1e-3
    assert abs(r["loss"] - g["loss"]) < 1e-3
    for k, d in g["grad_digest"].items():
        gk = r["grads"][k].double()
        assert abs(gk.sum().item() - d["sum"]) <= 2e-2 * d["abs"] + 1e-6, k
        assert abs((gk * gk).sum().item() - d["sq"]) <= 2e-2 * d["sq"] + 1e-9, k
    for key in ("running_1", "running_3"):
        for k, v in g[key].items():
            got = r[key][k]
            if v.dtype == torch.int64:
                assert torch.equal(got, v), k
            else:
                assert torch.allclose(got, v, rtol=1e-3, atol=1e-4), k
    assert rel_err(r["eval_1"], g["eval_logits_1"].float()) < 3e-3
    assert rel_err(r["eval_3"], g["eval_logits_3"].float()) < 3e-3


@pytest.mark.parametrize("name", ["unet2d_single", "unet2d_basic"])
def test_model_amp_close_to_reference(name):
    g = load_golden(name)
    cfg = g["cfg"]
    net = b200seg.UNet2D(1, cfg["classes"], cfg["base"], block=cfg["block"])
    net.load_state_dict(seeded_state_dict(net, cfg["state_seed"]))
    net = net.to(DEV)
    with torch.autocast("cuda", dtype=torch.float16):
        r = _run_steps(net, cfg, DEV)
    assert rel_err(r["logits"].float(), g["logits"]) < 3e-2
    assert abs(r["loss"] - g["loss"]) < 2e-2
    assert torch.equal(r["running_3"][[k for k in g["running_3"] if "num_batches" in k][0]],
                       g["running_3"][[k for k in g["running_3"] if "num_batches" in k][0]])


def _acdc_step(block, seed):
    torch.manual_seed(seed)
    net = b200seg.UNet2D(1, 4, 32, block=block).to(DEV)
    torch.manual_seed(seed)
    ema = b200seg.UNet2D(1, 4, 32, block=block).to(DEV)
    ema.load_state_dict(net.state_dict())
    opt = FusedAdamWEMA(net, ema, amp=True)
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.randn(32, 1, 256, 256, device=DEV, generator=g)
    lab = torch.randint(0, 4, (32, 1, 256, 256), device=DEV, generator=g)
    crit = b200seg.DiceCELoss(weight=torch.tensor([0.5, 1.0, 1.0, 1.0]))
    torch.cuda.reset_peak_memory_stats()
    net.train()
    opt.zero_grad()
    with torch.autocast("cuda", dtype=torch.float16):
        loss = crit(net(img), lab)
    opt.scale_loss(loss).backward()
    opt.step()
    torch.cuda.synchronize()
    return loss.item(), {k: v.detach().clone() for k, v in net.state_dict().items()}, \
        {k: v.detach().clone() for k, v in ema.state_dict().items()}, torch.cuda.max_memory_allocated()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("block", ["SingleConv", "BasicBlock"])
def test_acdc_fullsize_step(block):
    l1, s1, e1, peak = _acdc_step(block, 0)
    l2, s2, e2, _ = _acdc_step(block, 0)
    print("ACDC 2D %s B=32 256x256 AMP step: loss %.5f, peak memory %.2f GB" % (block, l1, peak / 2 ** 30))
    assert torch.isfinite(torch.tensor(l1))
    assert l1 == l2
    for k in s1:
        assert torch.equal(s1[k], s2[k]), k
        assert torch.equal(e1[k], e2[k]), k
    nbt = [k for k in e1 if k.endswith("num_batches_tracked")]
    assert all(int(e1[k]) == 1 for k in nbt)        # the EMA net's buffers are copied from the trained net


@pytest.mark.parametrize("block", ["SingleConv", "BasicBlock"])
@pytest.mark.parametrize("sliding", [False, True])
def test_inference_2d_matches_reference_functions(block, sliding):
    """get_inference(dimension='2d') on a [D,1,H,W] slice stack against inference/inference2d.py (restated in
    oracle/unet2d.py) run on the stock-torch oracle net with the same state_dict, both in eval mode."""
    import types
    from oracle import unet2d as oref
    net = b200seg.UNet2D(1, 4, 8, block=block)
    net.load_state_dict(seeded_state_dict(net, 11))
    ref = oref.UNet2DRef(1, 4, 8, block=block)
    ref.load_state_dict(net.state_dict())
    net, ref = net.to(DEV), ref.to(DEV)
    args = types.SimpleNamespace(dimension="2d", sliding_window=sliding, window_size=[64, 64], classes=4)
    g = torch.Generator().manual_seed(21)
    stack = torch.randn(6, 1, 96 if sliding else 64, 80 if sliding else 64, generator=g).to(DEV)
    ours = b200seg.get_inference(args)(net, stack, args)
    allow = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        want = (oref.inference_sliding_window if sliding else oref.inference_whole_image)(ref, stack, args)
    finally:
        torch.backends.cudnn.allow_tf32 = allow
    assert ours.shape == want.shape
    assert (ours - want).abs().max().item() < 1e-3
    assert torch.allclose(ours.sum(1), torch.ones_like(ours.sum(1)), atol=1e-5)
