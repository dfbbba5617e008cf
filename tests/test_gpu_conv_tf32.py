"""GPU: fp32 convolutions on TF32 tensor cores (ALGO_TC_TF32, conv_tc_kernel_tf32<NT, KSTEPS>), against float64.

Kernel level: every (NT, KSTEPS) instantiation, and every forward mode — raw input, InstanceNorm + ReLU / LeakyReLU in
the loader, the per-channel (BatchNorm) table, bias, residual — and the data-gradient mode with its activation mask and
both InstanceNorm-backward sums, on channel-sliced operands (ld / coff), volumes that are not tile multiples, kernels
1x1x1 / 1x3x3 / 3x3x3 and B > 1.  Each element must satisfy

    |y - y64| <= (2^-9 + K 2^-23) (|a| * |w|)64 |act'(h)|  +  2^-22 (|a| * |w| + |bias| + |res|)64

with a the loader-transformed input and K = Cin taps.  The first term is the GEMM: both operands rounded or truncated
to TF32 (at most 2^-10 relative each, 2^-9 for the product) and K fp32 additions; the second the fp32 roundings of the
bias add, the residual add and the store.  No tolerance is tuned.  The InstanceNorm sums must match fp64 sums of the
kernel's own y.

Model level: an eval forward in TF32 mode of ResUNet 3D, UNet2D (running statistics), UNETR (Linears) and MedFormer has a
normalised logit error against fp64 of at most twice that of the stock-torch oracle module on cuDNN / cuBLAS TF32 with
the same weights and input; so does one ResUNet fp32 training step (loss and gradients).  Switching TF32 off again gives
the exact path bit for bit, and sliding-window validation in TF32 mode keeps its probability error within twice cuDNN
TF32's and labels every voxel that error cannot flip as the exact path does.

Every test that turns TF32 on restores torch.backends.cuda.matmul.fp32_precision to exactly its saved value."""
import copy
import re
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import losses as olosses
from oracle import unet3d as ounet
from oracle.synth import make_volume
from util import global_l2, launched_kernels, load_golden, rel_err

pytestmark = pytest.mark.gpu

EPS = 1e-4
STATS_BAR = 1e-5
MASK_MARGIN = 1e-3
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2
NTS = (16, 32, 48, 64, 80, 96, 112, 128)
MODES = ("raw", "in_relu", "in_lrelu", "pc_relu", "bias", "res", "dgrad_relu", "dgrad_lrelu")


@pytest.fixture
def tf32():
    """turns TF32 on (torch's matmul precision) for one test; restores exactly the saved value, and cuDNN's conv flag
    (the oracle's TF32 switch) likewise"""
    saved = torch.backends.cuda.matmul.fp32_precision, torch.backends.cudnn.conv.fp32_precision
    torch.backends.cudnn.conv.fp32_precision = "tf32"

    def set_(on):
        torch.backends.cuda.matmul.fp32_precision = "tf32" if on else saved[0]
    yield set_
    torch.backends.cuda.matmul.fp32_precision, torch.backends.cudnn.conv.fp32_precision = saved


# ----------------------------------------------------------------------------- kernel level
def _rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def nc(t):
    return t.double().permute(0, 4, 1, 2, 3)


def stats64(t):
    d = t.double().flatten(1, 3)
    return torch.stack([d.sum(1), (d * d).sum(1)], -1).contiguous()


def xhat64(t, st):
    n = t[0, ..., 0].numel()
    m = st[..., 0] / n
    r = 1.0 / torch.sqrt((st[..., 1] / n - m * m).clamp_min(0) + EPS)
    return (nc(t) - m[:, :, None, None, None]) * r[:, :, None, None, None]


def act64(h, act):
    return h if act == ACT_NONE else (h.clamp_min(0) if act == ACT_RELU else torch.where(h > 0, h, 0.01 * h))


def dact64(h, act):
    one = torch.ones_like(h)
    return torch.where(h > 0, one, (0.0 if act == ACT_RELU else 0.01) * one)


def _row(Cin, Cout, k, shape, mode, ld_pad=0, coff=0):
    return (Cin, Cout, k, shape, mode, ld_pad, coff)


ROWS = {}
for _m in MODES:
    ROWS["k333_b2-" + _m] = _row(32, 48, (3, 3, 3), (2, 3, 20, 12), _m)
    ROWS["k133_sliced-" + _m] = _row(24, 64, (1, 3, 3), (1, 2, 37, 21), _m, ld_pad=12, coff=4)
    ROWS["k111_b3-" + _m] = _row(40, 32, (1, 1, 1), (3, 2, 9, 17), _m, ld_pad=8, coff=8)
    ROWS["nkc3_ntiles2-" + _m] = _row(96, 256, (3, 3, 3), (1, 3, 17, 10), _m)            # streamed weights
for _m in ("raw", "in_relu", "res", "dgrad_relu"):
    ROWS["cin80_cpasync-" + _m] = _row(80, 112, (3, 3, 3), (2, 2, 16, 8), _m, ld_pad=4, coff=4)   # Cin > 64: cp.async loader
    ROWS["d1-" + _m] = _row(16, 16, (3, 3, 3), (2, 1, 20, 12), _m)


def _inputs(Cin, Cout, k, shape, mode, ld_pad, coff, seed):
    B, D, H, W = shape
    taps = k[0] * k[1] * k[2]
    xl = _rand(B, D, H, W, Cin + ld_pad, seed=seed, scale=1.5)
    x = xl[..., coff:coff + Cin]
    inp = dict(xl=xl, x=x, coff=coff, w=_rand(Cout, Cin, *k, seed=seed + 1) / (Cin * taps) ** 0.5, xst=None, act=ACT_NONE,
               table=None, bias=None, resl=None, r_coff=0, dg=None, want_stats=True)
    if mode.startswith("in_"):
        inp.update(xst=stats64(x), act=ACT_RELU if mode == "in_relu" else ACT_LRELU)
    elif mode == "pc_relu":
        g = torch.Generator().manual_seed(seed + 2)
        s = torch.rand(Cin, generator=g) + 0.5
        s[::3] = -s[::3]
        inp.update(table=torch.stack([s, torch.randn(Cin, generator=g)], 1).contiguous().cuda(), act=ACT_RELU)
    elif mode == "bias":
        inp.update(bias=_rand(Cout, seed=seed + 3, scale=0.5), want_stats=False)
    elif mode == "res":
        inp.update(xst=stats64(x), act=ACT_RELU, resl=_rand(B, D, H, W, Cout + ld_pad, seed=seed + 4), r_coff=ld_pad)
    elif mode.startswith("dgrad"):
        gl = _rand(B, D, H, W, Cout + ld_pad, seed=seed + 5)
        gx = gl[..., ld_pad:]
        inp["dg"] = (gl, ld_pad, stats64(gx), ACT_RELU if mode == "dgrad_relu" else ACT_LRELU)
    else:
        assert mode == "raw", mode
    return inp


def _launch(inp, Cin, Cout, k):
    from b200seg import _lib, batchnorm, ops
    wp = ops.pack_weight(inp["w"], torch.float32, layout=_lib.ALGO_TC_TF32)
    if inp["table"] is not None:
        assert inp["coff"] == 0
        return batchnorm.conv_pc_fwd(inp["xl"], Cin, inp["table"], inp["act"], (wp, _lib.ALGO_TC_TF32), Cout, k,
                                     bias=inp["bias"], want_stats=inp["want_stats"])
    return ops.conv3d_fwd(inp["xl"], inp["coff"], Cin, inp["xst"], inp["act"], wp, Cout, k, bias=inp["bias"],
                          residual=inp["resl"], r_coff=inp["r_coff"], want_stats=inp["want_stats"], dgrad_of=inp["dg"],
                          algo=_lib.ALGO_TC_TF32)


def _check(inp, Cin, Cout, k, y, y_stats):
    """the per-element bound of the module docstring and the InstanceNorm sums; returns the largest |y - y64| / bound"""
    pad = [i // 2 for i in k]
    if inp["table"] is not None:
        a = act64(nc(inp["x"]) * inp["table"][:, 0].double()[:, None, None, None] + inp["table"][:, 1].double()[:, None, None, None], inp["act"])
    elif inp["xst"] is not None:
        a = act64(xhat64(inp["x"], inp["xst"]), inp["act"])
    else:
        a = nc(inp["x"])
    w64 = inp["w"].double()
    y64 = F.conv3d(a, w64, padding=pad)
    mag = F.conv3d(a.abs(), w64.abs(), padding=pad)
    K = Cin * k[0] * k[1] * k[2]
    gemm = (2.0 ** -9 + K * 2.0 ** -23) * mag
    extra = mag.clone()
    if inp["bias"] is not None:
        y64 = y64 + inp["bias"].double()[:, None, None, None]
        extra = extra + inp["bias"].double().abs()[:, None, None, None]
    if inp["resl"] is not None:
        r = nc(inp["resl"][..., inp["r_coff"]:inp["r_coff"] + Cout])
        y64, extra = y64 + r, extra + r.abs()
    keep = torch.ones_like(y64, dtype=torch.bool)
    h = None
    if inp["dg"] is not None:
        gl, gcoff, gst, ga = inp["dg"]
        h = xhat64(gl[..., gcoff:gcoff + Cout], gst)
        d = dact64(h, ga)
        y64, gemm = y64 * d, gemm * d
        keep = h.abs() >= MASK_MARGIN
    bound = (gemm + 2.0 ** -22 * extra).clamp_min(1e-300)        # 0 only where y64 = 0 = y (a masked or empty sum)
    yd = nc(y)
    ratio = torch.where(keep, (yd - y64).abs() / bound, torch.zeros_like(bound))
    worst = ratio.max().item()
    assert worst <= 1.0, "element %s exceeds the TF32 bound by %.2fx" % (tuple(torch.nonzero(ratio == ratio.max())[0].tolist()), worst)
    if not inp["want_stats"]:
        assert y_stats is None
        return worst
    if h is None:
        sref = stats64(y)
    else:
        sref = torch.stack([yd.sum((2, 3, 4)), (yd * h).sum((2, 3, 4))], -1)
    assert rel_err(y_stats, sref) < STATS_BAR
    return worst


@pytest.mark.parametrize("row", list(ROWS))
def test_tf32_conv_against_fp64(row):
    from b200seg import _lib, ops
    Cin, Cout, k, shape, mode, ld_pad, coff = ROWS[row]
    B = 1 if mode == "pc_relu" else shape[0]
    assert _lib.load().b200seg_conv3d_algo_tf32(Cin, Cout, *k, B) == _lib.ALGO_TC_TF32
    if mode == "pc_relu":
        ld_pad, coff = 0, 0
    inp = _inputs(Cin, Cout, k, shape, mode, ld_pad, coff, seed=sum(map(ord, row)))
    y, st = _launch(inp, Cin, Cout, k)
    torch.cuda.synchronize()
    worst = _check(inp, Cin, Cout, k, y, st)
    # the row is on TF32: the exact CUDA-core result differs
    wd = ops.pack_weight(inp["w"], torch.float32)
    if inp["table"] is None:
        yd, _ = ops.conv3d_fwd(inp["xl"], inp["coff"], Cin, inp["xst"], inp["act"], wd, Cout, k, bias=inp["bias"],
                               residual=inp["resl"], r_coff=inp["r_coff"], want_stats=False, dgrad_of=inp["dg"],
                               algo=_lib.ALGO_DIRECT)
        assert not torch.equal(y, yd)
    print("%s: worst |y - y64| / bound %.3f" % (row, worst))


_INST = re.compile(r"conv_tc_kernel_tf32(?:<\s*(?:\(int\))?\s*(\d+)\s*,\s*(?:\(int\))?\s*(\d+)\s*>|ILi(\d+)ELi(\d+)E)")


def launch_every_instantiation():
    """one launch per (NT, KSTEPS) = (Cout, Cin / 8), the modes cycling over the instantiations; returns
    {(NT, KSTEPS): (inputs, Cin, Cout, (y, y_stats))}"""
    out = {}
    for i, (nt, ks) in enumerate((nt, ks) for nt in NTS for ks in (1, 2, 3, 4)):
        mode = ("raw", "in_lrelu", "res", "dgrad_relu", "bias", "in_relu", "dgrad_lrelu")[i % 7]
        inp = _inputs(8 * ks, nt, (3, 3, 3), (2, 3, 20, 12), mode, 0, 0, seed=i)
        out[(nt, ks)] = (inp, 8 * ks, nt, _launch(inp, 8 * ks, nt, (3, 3, 3)))
    torch.cuda.synchronize()
    return out


def test_every_tf32_instantiation_launches():
    """the 32 launches of launch_every_instantiation name all 32 conv_tc_kernel_tf32<NT, KSTEPS>, and each result is
    within the bound.  The profiler records them in a process of its own (util.launched_kernels): a profiling session
    in this process would make later sessions of the same pytest run lose launches."""
    names = launched_kernels("test_gpu_conv_tf32", "launch_every_instantiation")
    seen = set()
    for n in names:
        if "conv_tc_kernel_tf32" not in n:
            continue
        m = _INST.search(n)
        assert m, n
        g = [int(v) for v in m.groups() if v is not None]
        seen.add((g[0], g[1]))
    runs = launch_every_instantiation()
    print("conv_tc_kernel_tf32 instantiations launched: %d of 32" % len(seen))
    assert seen == set(runs), sorted(set(runs) - seen)
    for inp, ci, co, (y, st) in runs.values():
        _check(inp, ci, co, (3, 3, 3), y, st)


# ----------------------------------------------------------------------------- model level
def _resunet():
    import b200seg
    cfg = load_golden("resunet_iso")["cfg"]
    net = b200seg.UNet(1, cfg["base"], scale=cfg["scale"], kernel_size=cfg["kernel"], num_classes=cfg["classes"],
                       block=cfg["block"], norm="in")
    sd = ounet.make_state_dict(ounet.unet_param_shapes(1, cfg["base"], cfg["classes"], cfg["kernel"], cfg["block"]),
                               seed=cfg["state_seed"])
    net.load_state_dict(sd)
    img, lab = make_volume(*cfg["shape"], cfg["classes"], seed=cfg["data_seed"])
    return net.cuda(), sd, cfg, img.cuda(), lab.cuda()


def _case_resunet():
    net, sd, cfg, img, _ = _resunet()

    def oracle(dt):
        return ounet.unet_forward({k: v.cuda().to(dt) for k, v in sd.items()}, img.to(dt), cfg["scale"], cfg["kernel"], cfg["block"])
    return net.eval(), img, oracle


def _case_unet2d():
    import b200seg
    from oracle import unet2d as oref
    from oracle.make_golden_unet2d import seeded_state_dict
    cfg = load_golden("unet2d_basic")["cfg"]
    net = b200seg.UNet2D(1, cfg["classes"], cfg["base"], block=cfg["block"])
    net.load_state_dict(seeded_state_dict(net, cfg["state_seed"]))
    ref = oref.UNet2DRef(1, cfg["classes"], cfg["base"], block=cfg["block"])
    ref.load_state_dict(net.state_dict())
    ref = ref.cuda().eval()
    B, H, W = cfg["shape"]
    img = _rand(B, 1, H, W, seed=cfg["data_seeds"][0])

    def oracle(dt):
        return copy.deepcopy(ref).to(dt)(img.to(dt))
    return net.cuda().eval(), img, oracle


def _case_unetr():
    import b200seg
    from oracle import unetr as ounetr
    g = load_golden("unetr_small")
    c = g["cfg"]
    net = b200seg.UNETR(c["in_ch"], c["classes"], c["size"], feature_size=c["feature_size"], hidden_size=c["hidden"],
                        mlp_dim=c["mlp"], num_heads=c["heads"])
    sd = ounetr.seeded_state_dict(g["shapes"], c["state_seed"])
    net.load_state_dict(sd)
    img, _ = make_volume(c["batch"], *c["size"], c["classes"], seed=c["data_seed"], in_ch=c["in_ch"])
    img = img.cuda()

    def oracle(dt):
        return ounetr.unetr_forward({k: v.cuda().to(dt) for k, v in sd.items()}, img.to(dt), c["heads"])
    return net.cuda().eval(), img, oracle


def _case_medformer():
    from oracle import medformer as omed
    from test_gpu_medformer import _build
    g = load_golden("medformer_bcv")
    cfg = g["cfg"]
    net, sd, kw = _build(g)
    img, _ = make_volume(*cfg["shape"], cfg["classes"], seed=cfg["data_seed"])
    img = img.cuda()

    def oracle(dt):
        r = omed.medformer_forward({k: v.cuda().to(dt) for k, v in sd.items()}, img.to(dt), kw)
        return r[0] if isinstance(r, (list, tuple)) else r
    return net.eval(), img, oracle


def _first(out):
    return out[0] if isinstance(out, (list, tuple)) else out


@pytest.mark.parametrize("model", ["resunet3d", "unet2d", "unetr", "medformer"])
def test_model_error_within_twice_cudnn_tf32(model, tf32):
    net, img, oracle = {"resunet3d": _case_resunet, "unet2d": _case_unet2d, "unetr": _case_unetr,
                        "medformer": _case_medformer}[model]()
    with torch.no_grad():
        ref64 = oracle(torch.float64).double()
        exact = _first(net(img)).detach().clone()
        tf32(True)
        ours = _first(net(img)).detach().clone()
        cud = oracle(torch.float32)
    e_ours, e_cudnn, e_exact = rel_err(ours, ref64), rel_err(cud, ref64), rel_err(exact, ref64)
    print("%s eval forward, normalised logit error vs fp64: b200seg TF32 %.2e, stock torch on cuDNN TF32 %.2e, "
          "b200seg exact fp32 %.2e" % (model, e_ours, e_cudnn, e_exact))
    assert not torch.equal(ours, exact)              # the TF32 kernels ran
    assert e_ours <= 2 * e_cudnn


def test_toggle_back_to_exact_is_bit_identical(tf32):
    net, _, _, img, _ = _resunet()
    net.eval()
    with torch.no_grad():
        a = net(img).clone()
        tf32(True)
        b = net(img).clone()
        tf32(False)
        c = net(img).clone()
    assert torch.equal(a, c)
    assert not torch.equal(a, b)


def test_sliding_window_labels_match_exact(tf32):
    """validation as the reference runs it (half-overlap windows, softmax average, argmax, Dice).  The averaged
    probabilities of the TF32 path are within twice the error of the stock-torch oracle's on cuDNN TF32 (both against
    fp64), and its label map is the exact path's at every voxel whose fp64 top-2 margin exceeds what the two paths'
    probability errors can move: 2 (e_tf32 + e_exact).  A fixed 1e-3 margin is no bar for TF32: on this volume cuDNN
    TF32 itself moves probabilities by 2e-2 and flips labels whose fp64 margin is 1.8e-2 (H100, see DESIGN.md 3.1)."""
    import b200seg
    from test_gpu_inference import _ref_sliding_window
    net, sd, cfg, _, _ = _resunet()
    img, lab = make_volume(1, 48, 40, 56, cfg["classes"], seed=31)
    img, lab = img.cuda(), lab.cuda()
    args = types.SimpleNamespace(window_size=[32, 32, 32], classes=cfg["classes"], dimension="3d", sliding_window=True)

    def oracle(dt):
        s = {k: v.cuda().to(dt) for k, v in sd.items()}
        return _ref_sliding_window(lambda x: ounet.unet_forward(s, x.to(dt), cfg["scale"], cfg["kernel"], cfg["block"]),
                                   img, args).double()
    p64 = oracle(torch.float64)
    top2 = p64.topk(2, dim=1).values
    margin = top2[:, 0] - top2[:, 1]
    p_exact, lab_exact = b200seg.inference_sliding_window(net, img, args, return_label=True)
    tf32(True)
    p_tf32, lab_tf32 = b200seg.inference_sliding_window(net, img, args, return_label=True)
    p_cudnn = oracle(torch.float32)
    e_exact, e_tf32, e_cudnn = ((p.double() - p64).abs().max().item() for p in (p_exact, p_tf32, p_cudnn))
    d_exact = b200seg.calculate_dice(lab_exact.reshape(-1, 1), lab.reshape(-1, 1), cfg["classes"])[0]
    d_tf32 = b200seg.calculate_dice(lab_tf32.reshape(-1, 1), lab.reshape(-1, 1), cfg["classes"])[0]
    differ = lab_exact != lab_tf32
    decided = margin > 2 * (e_tf32 + e_exact)
    print("sliding window: probability error vs fp64: exact %.2e, TF32 %.2e, cuDNN TF32 %.2e; %d of %d labels differ "
          "(%d where the fp64 margin exceeds 1e-3, largest such margin %.2e; %d where it exceeds %.2e); Dice exact %s, "
          "TF32 %s" % (e_exact, e_tf32, e_cudnn, differ.sum().item(), differ.numel(), (differ & (margin > 1e-3)).sum().item(),
                       margin[differ].max().item() if differ.any() else 0.0, (differ & decided).sum().item(),
                       2 * (e_tf32 + e_exact), d_exact.tolist(), d_tf32.tolist()))
    assert e_tf32 <= 2 * e_cudnn
    assert decided.float().mean().item() > 0.9
    assert not (differ & decided).any()
    assert torch.equal(lab_tf32.long(), p_tf32.argmax(1))


def test_resunet_training_step_within_twice_cudnn_tf32(tf32):
    """one fp32 training step in TF32 mode (the weight gradient stays on the exact path): loss and gradients against
    fp64, at most twice the error of the stock-torch oracle's step on cuDNN TF32"""
    import b200seg
    net, sd, cfg, img, lab = _resunet()
    w = torch.tensor(cfg["ce_weight"])

    def oracle(dt):
        s = {k: v.cuda().to(dt).requires_grad_(True) for k, v in sd.items()}
        lo = ounet.unet_forward(s, img.to(dt), cfg["scale"], cfg["kernel"], cfg["block"])
        loss = olosses.total_loss(lo, lab, w.cuda().to(dt))
        loss.backward()
        return loss.item(), {k: v.grad.double() for k, v in s.items()}
    l64, g64 = oracle(torch.float64)
    tf32(True)
    logits = net(img)
    loss = b200seg.DiceCELoss(weight=w)(logits, lab)
    loss.backward()
    ours = {k: p.grad.double() for k, p in net.named_parameters()}
    lc, gc = oracle(torch.float32)
    el, elc = abs(loss.item() - l64) / abs(l64), abs(lc - l64) / abs(l64)
    eg, egc = global_l2(ours, g64), global_l2(gc, g64)
    print("resunet TF32 training step vs fp64: loss %.2e (cuDNN TF32 %.2e), gradients global L2 %.2e (cuDNN TF32 %.2e)"
          % (el, elc, eg, egc))
    assert el <= 2 * max(elc, 2.0 ** -23)          # below fp32 resolution the two losses cannot be ranked
    assert eg <= 2 * egc
