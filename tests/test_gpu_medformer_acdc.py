"""GPU: the ACDC MedFormer configuration (config/acdc/medformer_3d.yaml: 2x6x6 = 72 map tokens, 4 heads per level ->
B-MHA at dim_head 32 / 64 / 80, map fusion over 3 x 72 tokens at dim_head 64) against float64.

  * the wide B-MHA entry (b200seg_biattn_wide_*): dim_head 32 / 64 / 80 at 72 tokens, ragged token counts, N tails of
    its 64-voxel blocks, heads 1 and 4, a peaked column softmax, the per-sample level shapes of the training crop, the raw
    ABI on channel-sliced operands, its refusals, and which entry BiAttnFn launches at ACDC and BCV shapes;
  * map generation at 72 and 80 codes, the dim_head 64 token attention up to 216 tokens;
  * the ACDC model against its reference fixture (tests/golden/medformer_acdc.pt) in fp32 and under AMP, and one full-size
    AMP TrainStep at 3 x 1 x 16 x 192 x 192.

Errors are max |got - ref| / max |ref| per output, held to the bars of tests/test_gpu_medformer_kernels.py."""
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import losses as olosses
from oracle import medformer as omed
from oracle import medformer_ops as mops
from oracle.synth import make_volume
from util import assert_untouched, global_l2, launched_kernels_each, load_golden, rel_err, sentinel, wide

pytestmark = pytest.mark.gpu

F16, F32 = torch.float16, torch.float32
DTYPES = [F32, F16]
DT_ID = {F32: "fp32", F16: "fp16"}
BARS = {"biattn": {F32: 1e-5, F16: 1.5e-3}, "mapgen": {F32: 3.5e-6, F16: 1.5e-3}, "mhsa": {F32: 6e-6, F16: 1.2e-3}}
SPECIAL_BARS = {"biattn": {F32: 8e-5, F16: 6e-3}, "mhsa": {F32: 8e-5, F16: 6e-3}}
WT = 64                  # voxels per block of the wide kernels


def _err(a, b):
    a, b = a.detach().double(), b.detach().double()
    scale = b.abs().max().item()
    return (a - b).abs().max().item() / (scale if scale > 0 else 1.0)


def _judge(kernel, tag, dtype, errs, special=False):
    print("ACDC_ERR %s %s %s %s" % (kernel, DT_ID[dtype], tag, {k: float("%.3e" % v) for k, v in errs.items()}))
    bar = (SPECIAL_BARS if special else BARS)[kernel][dtype]
    bad = {k: v for k, v in errs.items() if not v < bar}
    assert not bad, (tag, bad, bar)


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


@pytest.fixture(scope="module")
def lib():
    import b200seg  # noqa: F401
    from b200seg import _lib
    assert _lib.load().b200seg_check_device() == 0, "not an H100"
    return _lib


# ============================================================================================ wide B-MHA
def _biattn_inputs(B, N, M, heads, dh, dtype, seed, scale=1.5, peaked=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    inner = dh * heads
    fqv = _randn(g, B, N, 2 * inner, scale=scale)
    mqv = _randn(g, B, M, 2 * inner, scale=scale)
    if peaked:
        # token j's column maximum on one voxel of block (7 j) mod nblk, so the merge rescales across blocks
        nblk = (N + WT - 1) // WT
        fqv[..., :inner] *= 0.2
        for j in range(M):
            fqv[:, ((7 * j) % nblk) * WT + (j * 13) % WT, :inner] = 3.0 * mqv[:, j, :inner]
    return fqv.to(dtype), mqv.to(dtype), _randn(g, B, N, inner).to(dtype), _randn(g, B, M, inner).to(dtype)


def _biattn_reference(fqv, mqv, dfo, dmo, heads):
    f = fqv.double().requires_grad_(True)
    m = mqv.double().requires_grad_(True)

    def vol(t):
        return t.permute(0, 2, 1)[..., None, None]
    fo, mo = mops.bidirection_attention_core(*vol(f).chunk(2, 1), *vol(m).chunk(2, 1), heads)
    fo, mo = fo[..., 0, 0].permute(0, 2, 1), mo[..., 0, 0].permute(0, 2, 1)
    torch.autograd.backward([fo, mo], [dfo.double(), dmo.double()])
    return fo.detach(), mo.detach(), f.grad, m.grad


def _biattn_check(tag, B, N, M, heads, dh, dtype, seed, **kw):
    from b200seg.ops import BiAttnFn
    fqv, mqv, dfo, dmo = _biattn_inputs(B, N, M, heads, dh, dtype, seed, **kw)
    f, m = fqv.clone().requires_grad_(True), mqv.clone().requires_grad_(True)
    fo, mo = BiAttnFn.apply(f, m, heads, dh)
    torch.autograd.backward([fo, mo], [dfo, dmo])
    rfo, rmo, rdf, rdm = _biattn_reference(fqv, mqv, dfo, dmo, heads)
    inner = dh * heads
    errs = {"fo": _err(fo, rfo), "mo": _err(mo, rmo),
            "dfq": _err(f.grad[..., :inner], rdf[..., :inner]), "dfv": _err(f.grad[..., inner:], rdf[..., inner:]),
            "dmq": _err(m.grad[..., :inner], rdm[..., :inner]), "dmv": _err(m.grad[..., inner:], rdm[..., inner:])}
    _judge("biattn", tag, dtype, errs, special=kw.get("peaked", False))


# dim_head 32 / 64 / 80 at ACDC's 72 tokens, the ragged ends of the 80-row build (65, 80), fewer tokens at 64 / 80;
# N: one voxel, one short of / exactly / one past a 64-voxel block, and several blocks with a ragged tail
WIDE_ROWS = [(2, n, 72, h, dh) for dh in (32, 64, 80) for n, h in ((1, 4), (63, 1), (64, 4), (65, 1), (600, 4))]
WIDE_ROWS += [(2, 129, m, h, dh) for dh in (32, 64, 80) for m, h in ((65, 4), (80, 1))]
WIDE_ROWS += [(2, 300, m, h, 64) for m, h in ((1, 1), (27, 4), (64, 4))] + [(2, 200, 8, 4, 80)]
# the training crop's per-sample levels (16x192x192, map 2x6x6): down2 / up2, down3 / up1, down4
WIDE_LEVELS = [(1, 16 * 48 * 48, 72, 4, 32), (1, 8 * 24 * 24, 72, 4, 64), (1, 4 * 12 * 12, 72, 4, 80)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,N,M,heads,dh", WIDE_ROWS, ids=["B%d-N%d-M%d-h%d-dh%d" % r for r in WIDE_ROWS])
def test_biattn_wide(B, N, M, heads, dh, dtype):
    _biattn_check("B%d-N%d-M%d-h%d-dh%d" % (B, N, M, heads, dh), B, N, M, heads, dh, dtype, seed=N + 7 * M + heads + dh)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,N,M,heads,dh", WIDE_LEVELS, ids=["N%d-dh%d" % (r[1], r[4]) for r in WIDE_LEVELS])
def test_biattn_wide_acdc_levels(B, N, M, heads, dh, dtype):
    _biattn_check("level-N%d-dh%d" % (N, dh), B, N, M, heads, dh, dtype, seed=5 + dh)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_biattn_wide_peaked(dtype):
    _biattn_check("peaked72", 2, WT * 80, 72, 4, 64, dtype, seed=17, peaked=True)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("N,M,heads,dh", [(129, 72, 4, 32), (70, 80, 1, 80), (600, 27, 4, 64)])
def test_biattn_wide_abi_sliced_operands(lib, N, M, heads, dh, dtype):
    """Every operand a channel slice of a wider row: the packed call's numbers bit for bit, the other channels of the
    outputs untouched, and nothing written past b200seg_biattn_wide_workspace bytes."""
    from b200seg import ops
    from b200seg.ops import _dt, _stream
    B, inner = 2, dh * heads
    fqv, mqv, dfo, dmo = _biattn_inputs(B, N, M, heads, dh, dtype, seed=21)
    fo_p, mo_p, colstat_p = ops.biattn_wide_fwd(fqv, mqv, heads, dh)
    dfqv_p, dmqv_p = ops.biattn_wide_bwd(fqv, mqv, mo_p, colstat_p, dfo, dmo, heads, dh)
    fq, fv, dfo_w = wide(fqv[..., :inner], inner + 24, 8), wide(fqv[..., inner:], inner + 40, 24), wide(dfo, inner + 24, 16)
    mb = wide(torch.cat([mqv[..., :inner], torch.zeros_like(mqv[..., :8]), mqv[..., inner:]], -1), 2 * inner + 32, 8)
    dmo_w = wide(dmo, inner + 32, 24)
    fo, dfq, dfv = sentinel((B, N), inner + 48, dtype), sentinel((B, N), inner + 32, dtype), sentinel((B, N), inner + 32, dtype)
    mo, dm = sentinel((B, M), inner + 16, dtype), sentinel((B, M), 2 * inner + 16, dtype)
    colstat = torch.empty(B, heads, M, 2, device="cuda")
    nbytes = lib.load().b200seg_biattn_wide_workspace(B, N, M, heads, dh)
    ws = torch.empty(nbytes // 4 + 64, device="cuda")
    canary = torch.randn(64, device="cuda")
    ws[nbytes // 4:] = canary
    mld, mq_off, mv_off = mb.shape[-1], 8, 16 + inner
    lib.call("b200seg_biattn_wide_fwd", fq.data_ptr(), fq.shape[-1], 8, fv.data_ptr(), fv.shape[-1], 24,
             mb.data_ptr(), mq_off, mb.data_ptr(), mv_off, mld, fo.data_ptr(), fo.shape[-1], 40, mo.data_ptr(),
             mo.shape[-1], 8, colstat.data_ptr(), ws.data_ptr(), B, N, M, heads, dh, dh ** -0.5, _dt(fqv), _stream())
    lib.call("b200seg_biattn_wide_bwd", fq.data_ptr(), fq.shape[-1], 8, fv.data_ptr(), fv.shape[-1], 24,
             mb.data_ptr(), mq_off, mb.data_ptr(), mv_off, mld, mo.data_ptr(), mo.shape[-1], 8, colstat.data_ptr(),
             dfo_w.data_ptr(), dfo_w.shape[-1], 16, dmo_w.data_ptr(), dmo_w.shape[-1], 24,
             dfq.data_ptr(), dfq.shape[-1], 8, dfv.data_ptr(), dfv.shape[-1], 32,
             dm.data_ptr(), 16 + inner, dm.data_ptr(), 0, dm.shape[-1], ws.data_ptr(), B, N, M, heads, dh, dh ** -0.5,
             _dt(fqv), _stream())
    torch.cuda.synchronize()
    assert torch.equal(ws[nbytes // 4:], canary), "the kernels wrote past b200seg_biattn_wide_workspace bytes"
    for name, buf, coff, ref in (("fo", fo, 40, fo_p), ("mo", mo, 8, mo_p), ("dfq", dfq, 8, dfqv_p[..., :inner]),
                                 ("dfv", dfv, 32, dfqv_p[..., inner:])):
        assert torch.equal(buf[..., coff:coff + inner], ref), name
        assert_untouched(buf, coff, inner)
    assert torch.equal(dm[..., 16 + inner:16 + 2 * inner], dmqv_p[..., :inner])
    assert torch.equal(dm[..., :inner], dmqv_p[..., inner:])
    assert torch.equal(dm[..., inner:16 + inner], torch.full_like(dm[..., inner:16 + inner], -777.0))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_biattn_wide_refusals(lib, dtype):
    """The wide entry refuses what the original entry owns (dim_head 32 with <= 64 tokens), more than 80 tokens and
    head sizes it is not built for, so every shape has exactly one path."""
    from b200seg import ops
    for M, heads, dh in ((64, 2, 32), (27, 4, 32), (1, 1, 32), (81, 1, 64), (81, 4, 32), (8, 1, 128), (8, 1, 48)):
        f = torch.zeros(1, 70, 2 * dh * heads, dtype=dtype, device="cuda")
        m = torch.zeros(1, M, 2 * dh * heads, dtype=dtype, device="cuda")
        with pytest.raises(lib.B200SegError):
            ops.biattn_wide_fwd(f, m, heads, dh)
        mo, colstat = torch.zeros(1, M, dh * heads, dtype=dtype, device="cuda"), torch.ones(1, heads, M, 2, device="cuda")
        with pytest.raises(lib.B200SegError):
            ops.biattn_wide_bwd(f, m, mo, colstat, torch.zeros(1, 70, dh * heads, dtype=dtype, device="cuda"), mo, heads, dh)


def run_biattn(N, M, heads, dh):
    """BiAttnFn forward + backward in fp16 (for the kernel-launch record)"""
    from b200seg.ops import BiAttnFn
    f = torch.randn(1, N, 2 * heads * dh, device="cuda", dtype=F16, requires_grad=True)
    m = torch.randn(1, M, 2 * heads * dh, device="cuda", dtype=F16, requires_grad=True)
    fo, mo = BiAttnFn.apply(f, m, heads, dh)
    (fo.float().sum() + mo.float().sum()).backward()
    torch.cuda.synchronize()


def test_biattn_dispatch():
    """BiAttnFn launches the wide kernels at ACDC's shapes and the original ones at BCV's (27 tokens) and AMOS / KiTS'
    (64 tokens) at dim_head 32."""
    shapes = [(1000, 72, 4, 32), (1000, 72, 4, 64), (500, 72, 4, 80), (1000, 27, 4, 32), (1000, 64, 8, 32)]
    names = launched_kernels_each("test_gpu_medformer_acdc", [("run_biattn", s) for s in shapes])
    for (N, M, heads, dh), ks in zip(shapes, names):
        wide_k = [k for k in ks if "biattn_wide" in k]
        old_k = [k for k in ks if "biattn" in k and "biattn_wide" not in k]
        if dh == 32 and M <= 64:
            assert old_k and not wide_k, (M, dh, ks)
        else:
            assert len(wide_k) >= 4 and not old_k, (M, dh, ks)


# ============================================================================================ map generation
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,N,K,C", [(2, 1000, 72, 128), (2, 129, 72, 256), (1, 4608, 72, 320), (2, 300, 80, 128),
                                     (2, 1, 72, 8), (2, 127, 65, 48)])
def test_mapgen_80_codes(B, N, K, C, dtype):
    """72 and 80 codes (the 80-code build), the fused projection padded to 16 channels as SemanticMapGeneration pads
    it (72 codes at 128 / 256 / 320 channels: 8 padded logit columns, whose gradient must be exactly zero)."""
    from b200seg.medformer_ops import MapGenFn
    g = torch.Generator(device="cuda").manual_seed(N + K + C)
    pad = (-(C + K)) % 16
    fw = _randn(g, B, N, C + K + pad, scale=1.5)
    fw[..., C + K:] = 0
    fw = fw.to(dtype)
    f64 = fw.double().requires_grad_(True)
    ref = torch.einsum("bnc,bnk->bkc", f64[..., :C], F.softmax(f64[..., C:C + K], dim=1))
    gm = _randn(g, B, K, C).to(dtype)
    ref.backward(gm.double())
    x = fw.clone().requires_grad_(True)
    smap = MapGenFn.apply(x, C, K, (1, 1, K))
    smap.backward(gm.view(B, 1, 1, K, C))
    errs = {"map": _err(smap.view(B, K, C), ref), "dfeat": _err(x.grad[..., :C], f64.grad[..., :C]),
            "dlogit": _err(x.grad[..., C:C + K], f64.grad[..., C:C + K])}
    if pad:
        assert torch.count_nonzero(x.grad[..., C + K:]) == 0, "logit padding columns must get zero gradient"
    _judge("mapgen", "B%d-N%d-K%d-C%d" % (B, N, K, C), dtype, errs)


# ============================================================================================ MHSA, dim_head 64
def _mhsa_check(tag, B, L, heads, dtype, seed, scale=1.0):
    from b200seg.medformer_ops import MHSAFn
    g = torch.Generator(device="cuda").manual_seed(seed)
    inner = 64 * heads
    qkv = _randn(g, B, L, 3 * inner, scale=scale).to(dtype)
    dout = _randn(g, B, L, inner).to(dtype)
    x = qkv.clone().requires_grad_(True)
    out = MHSAFn.apply(x, heads, 64)
    out.backward(dout)
    q64 = qkv.double().requires_grad_(True)
    q, k, v = (t.reshape(B, L, heads, -1).permute(0, 2, 1, 3) for t in q64.chunk(3, dim=-1))
    att = F.softmax(torch.einsum("bhid,bhjd->bhij", q, k) * 64 ** -0.5, dim=-1)
    ref = torch.einsum("bhij,bhjd->bhid", att, v).permute(0, 2, 1, 3).reshape(B, L, -1)
    ref.backward(dout.double())
    errs = {"out": _err(out, ref)}
    for i, nm in enumerate(("dq", "dk", "dv")):
        errs[nm] = _err(x.grad[..., i * inner:(i + 1) * inner], q64.grad[..., i * inner:(i + 1) * inner])
    _judge("mhsa", tag, dtype, errs, special=scale > 1.0)


MH64_ROWS = [(1 + (a + b) % 2, l, h) for a, l in enumerate([1, 64, 72, 144, 216]) for b, h in enumerate([1, 4])]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,L,heads", MH64_ROWS, ids=["B%d-L%d-h%d" % r for r in MH64_ROWS])
def test_mhsa_dh64(B, L, heads, dtype):
    _mhsa_check("dh64-B%d-L%d-h%d" % (B, L, heads), B, L, heads, dtype, seed=L * 16 + heads + B)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_mhsa_dh64_large_logit(dtype):
    _mhsa_check("dh64-large_logit", 2, 216, 4, dtype, seed=43, scale=3.0)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_mhsa_dh64_refuses_217_tokens(lib, dtype):
    from b200seg.medformer_ops import MHSAFn
    with pytest.raises(lib.B200SegError):
        MHSAFn.apply(torch.zeros(1, 217, 3 * 64, dtype=dtype, device="cuda"), 1, 64)


# ============================================================================================ whole model
def _build(g):
    import b200seg
    from oracle.unet3d import make_state_dict
    cfg = g["cfg"]
    kw = {k: cfg[k] for k in ("map_size", "conv_num", "trans_num", "num_heads", "fusion_depth", "fusion_dim",
                              "fusion_heads", "kernel_size", "scale", "aux_loss")}
    net = b200seg.MedFormer(1, cfg["classes"], 32, conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0,
                            proj_type="depthwise", norm="in", act="relu", **kw)
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == g["shapes"]
    sd = make_state_dict(g["shapes"], seed=cfg["state_seed"])
    for k in sd:
        if k.endswith("norm.weight"):
            sd[k] = 1.0 + 0.1 * sd[k] / sd[k].abs().max()
    net.load_state_dict(sd)
    return net.cuda(), sd, kw


def _oracle(sd, img, lab, w, aux_w, kw, dt=torch.float64):
    s = {k: v.to(dt).clone().requires_grad_(True) for k, v in sd.items()}
    r = omed.medformer_forward(s, img.to(dt), kw)
    olosses.total_loss(r, lab, w.to(dt), aux_w).backward()
    return {k: v.grad.double() for k, v in s.items()}, [t.detach().double() for t in r]


def _our_loss(b200seg, res, lab, w, aux_w):
    crit = b200seg.DiceCELoss(weight=w)
    return sum(aux_w[j] * crit(r, lab) for j, r in enumerate(res))


def test_medformer_acdc_fp32_matches_reference():
    """The fixture of the unmodified reference (logits, argmax, loss) and the float64 oracle's gradients, with the bars
    of test_medformer_fp32_matches_reference."""
    import b200seg
    g = load_golden("medformer_acdc")
    cfg = g["cfg"]
    net, sd, kw = _build(g)
    img, lab = make_volume(*cfg["shape"], cfg["classes"], seed=cfg["data_seed"])
    w = torch.tensor(cfg["ce_weight"])
    res = net(img.cuda())
    loss = _our_loss(b200seg, res, lab.cuda(), w, cfg["aux_weight"])
    loss.backward()
    for o, ref, am in zip(res, g["logits"], g["argmax"]):
        lg = o.detach().float().cpu()
        assert lg.shape == ref.shape
        assert rel_err(lg, ref.float()) < 2e-3
        assert (lg.argmax(1).to(torch.uint8) == am).float().mean().item() > 0.9995
    assert abs(loss.item() - g["loss"]) < 1e-4
    g64, l64 = _oracle(sd, img, lab, w, cfg["aux_weight"], kw)
    g32, _ = _oracle(sd, img, lab, w, cfg["aux_weight"], kw, torch.float32)
    for o, ref in zip(res, l64):
        assert rel_err(o.detach().float().cpu(), ref) < 1e-3
    ours = {k: p.grad for k, p in net.named_parameters()}
    floor, err = global_l2(g32, g64), global_l2(ours, g64)
    gmax = max(v.abs().max().item() for v in g64.values())
    worst = max(((ours[k].double().cpu() - g64[k]).abs().max() / (g64[k].abs().max() + 1e-4 * gmax)).item() for k in g64)
    floor_w = max(((g32[k] - g64[k]).abs().max() / (g64[k].abs().max() + 1e-4 * gmax)).item() for k in g64)
    print("medformer_acdc: global L2 grad err %.2e (reference fp32 floor %.2e); worst tensor %.2e (floor %.2e)"
          % (err, floor, worst, floor_w))
    assert err < max(1e-3, 3 * floor)
    assert worst < max(2e-3, 6 * floor_w)


def test_medformer_acdc_amp_close_to_fp32_reference():
    import b200seg
    g = load_golden("medformer_acdc")
    cfg = g["cfg"]
    net, sd, kw = _build(g)
    img, lab = make_volume(*cfg["shape"], cfg["classes"], seed=cfg["data_seed"])
    w = torch.tensor(cfg["ce_weight"])
    scale = 1024.0
    with torch.autocast("cuda", dtype=torch.float16):
        res = net(img.cuda())
        assert res[0].dtype == torch.float16
        loss = _our_loss(b200seg, res, lab.cuda(), w, cfg["aux_weight"])
    (loss * scale).backward()
    g64, l64 = _oracle(sd, img, lab, w, cfg["aux_weight"], kw)
    ours = {k: p.grad / scale for k, p in net.named_parameters()}
    err = global_l2(ours, g64)
    sdg = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.float16):
        rref = omed.medformer_forward(sdg, img.cuda(), kw)
        lref = olosses.total_loss(rref, lab.cuda(), w.cuda(), cfg["aux_weight"])
    (lref * scale).backward()
    amp_floor = global_l2({k: v.grad / scale for k, v in sdg.items()}, g64)
    e_ours = max(rel_err(o.detach().float().cpu(), r) for o, r in zip(res, l64))
    e_amp = max(rel_err(o.detach().float().cpu(), r) for o, r in zip(rref, l64))
    print("medformer_acdc amp: logits err ours %.2e | stock autocast %.2e ; global L2 grad err ours %.2e | stock "
          "autocast %.2e" % (e_ours, e_amp, err, amp_floor))
    assert e_ours < max(3e-2, 2 * e_amp)
    assert abs(loss.item() - g["loss"]) < max(3e-2, 2 * abs(lref.item() - g["loss"]))
    assert err < max(0.05, 2 * amp_floor)


ACDC = dict(map_size=[2, 6, 6], conv_num=[2, 0, 0, 0, 0, 0, 2, 2], trans_num=[0, 2, 2, 2, 2, 2, 0, 0],
            num_heads=[1, 4, 4, 4, 4, 4, 1, 1], fusion_depth=2, fusion_dim=256, fusion_heads=4,
            kernel_size=[[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
            scale=[[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2]], aux_loss=True)
AUX_WEIGHT = [0.5, 0.5]


def acdc_args():
    """get_model's arguments with the values of config/acdc/medformer_3d.yaml"""
    c = dict(ACDC)
    return types.SimpleNamespace(dimension="3d", model="medformer", in_chan=1, classes=4, base_chan=32,
                                 conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0, proj_type="depthwise",
                                 norm="in", act="relu", down_scale=c.pop("scale"), **c)


def _acdc_state(net):
    """seeded weights damped as test_gpu_medformer_kernels._bcv_state damps them, so fp16 rounding moves the logits by
    ~1e-2 instead of throwing a 36 864-voxel softmax into its chaotic regime"""
    from oracle.unet3d import make_state_dict
    sd = make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=7)
    damp = {"semantic_proj.weight": 0.1, "map_qv.weight": 0.3, "feat_qv.pointwise.weight": 0.3,
            "feedforward.pointwise.conv.weight": 0.2, "attn.feat_out.pointwise.weight": 0.2, "attn.map_out.weight": 0.2,
            "fn.to_out.weight": 0.2, "fn.fc2.weight": 0.2}
    for k, v in sd.items():
        if k.endswith("norm.weight"):
            sd[k] = 1.0 + 0.1 * v / v.abs().max()
        elif v.dim() == 1:
            sd[k] = 0.1 * v / v.abs().max()
        else:
            sd[k] = v * next((f for suffix, f in damp.items() if k.endswith(suffix)), 1.0)
    return sd


def test_fullsize_acdc_amp_trainstep():
    """One AMP TrainStep of get_model's ACDC MedFormer at the reference README's crop (3 x 1 x 16 x 192 x 192, 4
    classes, aux head): finite loss, every parameter updated, and its forward against the fp32 oracle on the GPU with
    stock autocast of the same oracle as the fp16 noise floor."""
    import b200seg
    from b200seg.train import TrainStep
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        args = acdc_args()
        net = b200seg.get_model(args)
        sd = _acdc_state(net)
        img, lab = make_volume(3, 16, 192, 192, 4, seed=2026)
        img, lab = img.cuda(), lab.cuda()
        w = torch.tensor([0.5, 1.0, 1.0, 1.0])
        with torch.no_grad():
            s = {k: v.cuda() for k, v in sd.items()}
            l32 = [t.double().cpu() for t in omed.medformer_forward(s, img, ACDC)]
            with torch.autocast("cuda", dtype=torch.float16):
                l_st = [t.double().cpu() for t in omed.medformer_forward(s, img, ACDC)]
            del s
        torch.cuda.empty_cache()
        net.load_state_dict(sd)
        net = net.cuda()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            lg = [t.double().cpu() for t in net(img)]
        e = max(rel_err(a, b) for a, b in zip(lg, l32))
        e_st = max(rel_err(a, b) for a, b in zip(l_st, l32))
        ema = b200seg.get_model(args)
        ema.load_state_dict(sd)
        ema = ema.cuda()
        step = TrainStep(net, ema, ce_weight=w, amp=True, aux_weight=AUX_WEIGHT)
        step.fused.scale.fill_(1024.0)
        loss = step(img, lab).item()
        torch.cuda.synchronize()
        moved = [k for k, p in net.named_parameters() if not torch.equal(p.detach().cpu(), sd[k])]
        print("medformer acdc 3x16x192x192 AMP: logits rel err vs fp32 oracle %.2e (stock autocast %.2e); loss %.5f; "
              "%d of %d parameter tensors updated" % (e, e_st, loss, len(moved), len(sd)))
        assert torch.isfinite(torch.tensor(loss))
        assert len(moved) == len(list(net.parameters()))
        assert e < max(5e-2, 3 * e_st)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
