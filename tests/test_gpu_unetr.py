"""GPU: UNETR path.
  * the global-attention kernels (csrc/attention.cu), fp16 tensor-core and fp32 CUDA-core, forward and backward,
    against an fp64 torch statement of monai's SABlock core at the configs' token counts (bcv / kits / lits 96^3:
    L = 216, acdc 16x192x192: L = 144, a 128^3 crop: L = 512) and at tile tails; bit-identical repeated backward;
  * one ViT TransformerBlock against the oracle;
  * the whole UNETR on the reference fixture (oracle/make_golden_unetr.py), with and without AMP;
  * the get_model configuration at 96^3, 14 classes, B = 2: one AMP step against the fp32 oracle, and two identical
    training steps through TrainStep / FusedAdamWEMA giving bit-identical parameters (LayerNorm affine parameters
    excepted, see the test)."""
import types

import pytest
import torch

from oracle import losses as olosses
from oracle import unetr as ounetr
from oracle.synth import make_volume
from util import global_l2, load_golden, rel_err

pytestmark = pytest.mark.gpu

ATTN_SHAPES = [(2, 216, 12), (1, 144, 12), (1, 512, 12), (2, 1, 2), (2, 27, 2), (1, 125, 3), (2, 200, 2)]


def _attn_inputs(B, L, heads, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, L, 3 * heads * 64, generator=g) * 1.5
    dout = torch.randn(B, L, heads * 64, generator=g)
    return qkv, dout


def _attn(qkv, dout, heads, dtype):
    from b200seg.unetr import AttentionFn
    x = qkv.cuda().to(dtype).requires_grad_(True)
    y = AttentionFn.apply(x, qkv.shape[0], heads)
    y.backward(dout.cuda().to(dtype))
    return y.detach(), x.grad.detach()


@pytest.mark.parametrize("B,L,heads", ATTN_SHAPES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_attention_matches_fp64(B, L, heads, dtype):
    qkv, dout = _attn_inputs(B, L, heads, seed=L * 10 + heads)
    qkv = qkv.to(dtype).float()                  # the exact answer for the inputs the kernel sees
    dout = dout.to(dtype).float()
    y, dq = _attn(qkv, dout, heads, dtype)
    x64 = qkv.double().cuda().requires_grad_(True)
    y64 = ounetr.sa_core(x64, heads)
    y64.backward(dout.double().cuda())
    e_y, e_dq = rel_err(y, y64), rel_err(dq, x64.grad)
    C = heads * 64
    g64 = x64.grad.cpu()
    floor = 1e-3 * g64.abs().max().item()        # dq = dk = 0 exactly at L = 1: measure those against the dv scale
    e_parts = [((dq[..., i * C:(i + 1) * C].double().cpu() - g64[..., i * C:(i + 1) * C]).abs().max()
                / max(g64[..., i * C:(i + 1) * C].abs().max().item(), floor)).item() for i in range(3)]
    print("attention B=%d L=%d heads=%d %s: out %.2e, dqkv %.2e (dq %.2e dk %.2e dv %.2e)"
          % (B, L, heads, dtype, e_y, e_dq, *e_parts))
    tol = (2e-5, 1e-4) if dtype == torch.float32 else (5e-3, 2e-2)
    assert e_y < tol[0]
    assert max(e_parts) < tol[1]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_attention_backward_is_deterministic(dtype):
    qkv, dout = _attn_inputs(2, 216, 12, seed=3)
    y1, d1 = _attn(qkv, dout, 12, dtype)
    y2, d2 = _attn(qkv, dout, 12, dtype)
    assert torch.equal(y1, y2) and torch.equal(d1, d2)


def test_attention_rejects_other_head_sizes():
    import b200seg
    from b200seg.unetr import AttentionFn
    x = torch.randn(1, 16, 3 * 4 * 32, device="cuda")
    with pytest.raises(b200seg.B200SegError, match="not supported"):
        AttentionFn.apply(x, 1, 4)


def _block_params(hidden, mlp, seed):
    from oracle.unet3d import make_state_dict
    shapes = {"mlp.linear1.weight": (mlp, hidden), "mlp.linear1.bias": (mlp,), "mlp.linear2.weight": (hidden, mlp),
              "mlp.linear2.bias": (hidden,), "norm1.weight": (hidden,), "norm1.bias": (hidden,),
              "attn.out_proj.weight": (hidden, hidden), "attn.out_proj.bias": (hidden,), "attn.qkv.weight": (3 * hidden, hidden),
              "norm2.weight": (hidden,), "norm2.bias": (hidden,)}
    sd = make_state_dict(shapes, seed=seed)
    for k in ("norm1.weight", "norm2.weight"):
        sd[k] = 1.0 + 0.1 * sd[k] / sd[k].abs().max()
    return sd


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_transformer_block_matches_oracle(dtype):
    from b200seg.unetr import TransformerBlock, _flat
    B, L, hidden, mlp, heads = 2, 216, 768, 3072, 12
    sd = _block_params(hidden, mlp, seed=21)
    blk = TransformerBlock(hidden, mlp, heads)
    blk.load_state_dict(sd)
    blk = blk.cuda()
    g = torch.Generator().manual_seed(22)
    x = torch.randn(B, L, hidden, generator=g)
    gy = torch.randn(B, L, hidden, generator=g)
    xt = x.cuda().to(dtype).view(*_flat(B * L), hidden).requires_grad_(True)
    y = blk(xt, B)
    y.backward(gy.cuda().to(dtype).view(*_flat(B * L), hidden))
    s64 = {k: v.double().cuda().requires_grad_(True) for k, v in sd.items()}
    x64 = x.to(dtype).double().cuda().requires_grad_(True)
    y64 = ounetr.transformer_block(s64, "", x64, heads)
    y64.backward(gy.to(dtype).double().cuda())
    errs = {k: rel_err(p.grad, s64[k].grad) for k, p in blk.named_parameters()}
    errs["x"] = rel_err(xt.grad.view(B, L, hidden), x64.grad)
    e = rel_err(y.view(B, L, hidden), y64)
    print("transformer block %s: out %.2e, grads %s" % (dtype, e, {k: "%.1e" % v for k, v in errs.items()}))
    tol = 1e-4 if dtype == torch.float32 else 1e-2
    assert e < tol
    assert max(errs.values()) < tol * 5, errs


def _small(amp):
    import b200seg
    g = load_golden("unetr_small")
    c = g["cfg"]
    net = b200seg.UNETR(c["in_ch"], c["classes"], c["size"], feature_size=c["feature_size"], hidden_size=c["hidden"],
                        mlp_dim=c["mlp"], num_heads=c["heads"])
    sd = ounetr.seeded_state_dict(g["shapes"], c["state_seed"])
    net.load_state_dict(sd)
    net = net.cuda()
    img, lab = make_volume(c["batch"], *c["size"], c["classes"], seed=c["data_seed"], in_ch=c["in_ch"])
    w = torch.tensor(c["ce_weight"])
    S = 1024.0 if amp else 1.0
    with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
        logits = net(img.cuda())
        loss = b200seg.DiceCELoss(weight=w)(logits, lab.cuda())
    (loss * S).backward()
    return g, c, sd, img, lab, w, net, logits, loss, S


@pytest.mark.parametrize("amp", [False, True])
def test_unetr_forward_backward(amp):
    g, c, sd, img, lab, w, net, logits, loss, S = _small(amp)
    lg = ounetr.voxel_sample(logits.detach().float().cpu(), g["stride"])     # the voxels the fixture stores
    e = rel_err(lg, g["logits"].float())
    agree = (lg.argmax(1).to(torch.uint8) == g["argmax"]).float().mean().item()
    so = {k: v.double().cuda().requires_grad_(True) for k, v in sd.items()}
    lo = ounetr.unetr_forward(so, img.double().cuda(), c["heads"])
    olosses.total_loss(lo, lab.cuda(), w.double().cuda()).backward()
    g64 = {k: v.grad.cpu() for k, v in so.items()}
    ours = {k: (p.grad / S).double().cpu() for k, p in net.named_parameters()}
    assert set(ours) == set(g64)
    l2 = global_l2(ours, g64)
    worst = sorted(((rel_err(ours[k], g64[k]), k) for k in g64), reverse=True)[:4]
    print("unetr amp=%d: logits rel err %.2e, label agreement %.5f, loss %.5f (ref %.5f), grads global-L2 %.2e, worst %s"
          % (amp, e, agree, loss.item(), g["loss"], l2, [(k, "%.1e" % v) for v, k in worst]))
    if amp:
        assert e < 5e-2 and agree > 0.97 and abs(loss.item() - g["loss"]) < 3e-2 and l2 < 0.25
    else:
        assert e < 2e-3 and agree > 0.9995 and abs(loss.item() - g["loss"]) < 1e-4 and l2 < 5e-3


BCV = dict(dimension="3d", model="unetr", in_chan=1, classes=14, training_size=[96, 96, 96])


def test_fullsize_amp_step():
    """get_model's UNETR at the bcv crop: an AMP forward/backward against the fp32 oracle (with stock torch autocast
    of the same oracle as the fp16 noise floor), then two identical TrainStep steps (fused AdamW + EMA) from the same
    state give the same loss and bit-identical parameters and EMA parameters."""
    import b200seg
    from b200seg.train import TrainStep
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        args = types.SimpleNamespace(**BCV)
        shapes = ounetr.unetr_param_shapes(1, 14, (96, 96, 96))
        sd = ounetr.seeded_state_dict(shapes, 7)
        img, lab = make_volume(2, 96, 96, 96, 14, seed=2024)
        img, lab = img.cuda(), lab.cuda()
        w = torch.tensor([0.5] + [1.0] * 13)

        def oracle(autocast, S):
            s = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                lo = ounetr.unetr_forward(s, img, 12)
                loss = olosses.total_loss(lo, lab, w.cuda())
            (loss * S).backward()
            return lo.detach().double().cpu(), loss.item(), {k: (v.grad / S).double().cpu() for k, v in s.items()}
        l32, loss32, g32 = oracle(False, 1.0)
        l_st, _, g_st = oracle(True, 1024.0)
        torch.cuda.empty_cache()

        net = b200seg.get_model(args)
        net.load_state_dict(sd)
        net = net.cuda()
        S = 1024.0
        with torch.autocast("cuda", dtype=torch.float16):
            logits = net(img)
            loss = b200seg.DiceCELoss(weight=w)(logits, lab)
        (loss * S).backward()
        lg = logits.detach().double().cpu()
        ours = {k: (p.grad / S).double().cpu() for k, p in net.named_parameters()}
        e, e_st = rel_err(lg, l32), rel_err(l_st, l32)
        l2, l2_st = global_l2(ours, g32), global_l2(g_st, g32)
        agree = (lg.argmax(1) == l32.argmax(1)).float().mean().item()
        print("unetr bcv AMP: logits rel err vs fp32 oracle %.2e (stock autocast %.2e); loss %.5f (oracle %.5f); grads "
              "global-L2 %.2e (stock autocast %.2e); label agreement %.5f" % (e, e_st, loss.item(), loss32, l2, l2_st, agree))
        assert e < max(5e-2, 3 * e_st)
        assert abs(loss.item() - loss32) < 2e-2
        assert l2 < max(0.1, 3 * l2_st)
        assert agree > 0.97
        del net, logits, loss, ours
        torch.cuda.empty_cache()

        def one_step():
            n = b200seg.get_model(args)
            n.load_state_dict(sd)
            n = n.cuda()
            ema = b200seg.get_model(args)
            ema.load_state_dict(sd)
            ema = ema.cuda()
            step = TrainStep(n, ema, ce_weight=w, amp=True)
            step.fused.scale.fill_(1024.0)      # a first step at GradScaler's 65536 may overflow in fp16 and be skipped
            lv = step(img, lab)
            torch.cuda.synchronize()
            return lv.item(), [p.detach().cpu() for p in n.parameters()], [p.detach().cpu() for p in ema.parameters()]
        la, pa, ea = one_step()
        torch.cuda.empty_cache()
        lb, pb, eb = one_step()
        moved = sum(1 for p, k in zip(pa, sd) if not torch.equal(p, sd[k]))
        differ = [k for k, x, y, u, v in zip(sd, pa, pb, ea, eb) if not (torch.equal(x, y) and torch.equal(u, v))]
        print("unetr bcv TrainStep: loss %.6f / %.6f, %d of %d parameter tensors updated; differing between the two "
              "runs: %s" % (la, lb, moved, len(pa), differ))
        assert la == lb
        assert moved > len(pa) // 2
        # LayerNormFn's backward (shared with MedFormer and SwinUNETR) sums d(gamma) / d(beta) with float atomics, so
        # only the LayerNorm affine parameters may differ in their last bits; everything else is bit-identical
        assert all(".norm" in k and k.split(".")[-1] in ("weight", "bias") for k in differ), differ
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
