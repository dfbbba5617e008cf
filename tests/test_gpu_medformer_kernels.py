"""GPU: the MedFormer kernels (csrc/biattn.cu, csrc/medformer_small.cu, csrc/dwconv.cu) against float64, at the shapes,
dtypes and edges where they can go wrong, and the benchmarked MedFormer (`medformer_bcv_96`) end to end.

  * B-MHA: the 32- and 64-row builds, every head count the configurations use, N tails and merge partitions that are
    empty or ragged, a column softmax whose maxima sit in different blocks and merge partitions, large logits, and the
    benchmark's level shapes (N = 96*24*24, 48*12*12, 24*6*6); the raw ABI on channel-sliced operands; refusals;
  * map generation, the 81-token MHSA, LayerNorm, GELU, the SE gate with the channel scale, space-to-depth and the
    depthwise convolution (with its fused InstanceNorm sums and weight gradient) at edge and benchmark shapes;
  * a recorded AMP step of the benchmarked MedFormer: every shape it sends to these kernels is in the tables below;
  * the benchmarked MedFormer at 96^3: an AMP step against the fp32 oracle, and two identical TrainSteps.

The reference is PyTorch float64 on the kernel's own (fp16-rounded) inputs.  Every output is judged on its own:
max |got - ref| over max |ref|, so an error confined to one tensor, one head or one third of a packed gradient cannot
hide under a larger neighbour."""
import json
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import losses as olosses
from oracle import medformer as omed
from oracle import medformer_ops as mops
from oracle import unet3d as ounet
from oracle.synth import make_volume
from util import global_l2, rel_err

pytestmark = pytest.mark.gpu

F16, F32 = torch.float16, torch.float32
DTYPES = [F32, F16]
DT_ID = {F32: "fp32", F16: "fp16"}

# Bars: the largest error measured over this file on an H100 80GB HBM3 (SXM, 700 W power limit), with at most 3x
# headroom (DESIGN.md §4 lists the rows that set them).  kernel -> dtype -> bar for every output of that kernel:
#              fp32                               fp16
#   biattn     3.4e-6 B2-N384-M27-h8 dfv          6.0e-4 B2-N128-M1-h8 dfq      (bench levels: 2.4e-6 / 4.5e-4)
#   mapgen     1.2e-6 B2-N129-K27-C320 dlogit     5.0e-4 B2-N127-K32-C56 dlogit (bench levels: 1.0e-6 / 3.8e-4)
#   mhsa       2.1e-6 large_logit out             4.5e-4 (output rounding)
#   layernorm  1.4e-5 offset300 dgamma            4.2e-4 (output rounding)
#   gelu       9.6e-8                             4.5e-4 (output rounding)
#   se         1.1e-6 C1280 d(excitation.2.w)     4.2e-4 (output rounding)
#   dwconv     8.3e-7 96x48x48 C128 dw            4.5e-4 (output rounding)
#   dwconv fused sums against the sums of the stored output: 5.3e-8
# The B-MHA and map-generation rows built to stress the softmax (a column maximum on one voxel per token, large
# logits) amplify fp rounding through exp and are held to SPECIAL_BARS instead, so the bench-level rows -- where the
# backward's c_j comes from the stored fp16 map output -- keep a bar within 3.3x of what they measure:
#   biattn     2.8e-5 large_logit dfv             2.6e-3 peaked64 dmq
#   mapgen     7.0e-6 peaked dlogit               1.7e-3 peaked dlogit
BARS = {
    "biattn": {F32: 1e-5, F16: 1.5e-3},
    "mapgen": {F32: 3.5e-6, F16: 1.5e-3},
    "mhsa": {F32: 6e-6, F16: 1.2e-3},
    "layernorm": {F32: 4e-5, F16: 1.2e-3},
    "gelu": {F32: 2.5e-7, F16: 1.2e-3},
    "se": {F32: 3e-6, F16: 1.2e-3},
    "dwconv": {F32: 2.4e-6, F16: 1.2e-3},
}
SPECIAL_BARS = {
    "biattn": {F32: 8e-5, F16: 6e-3},
    "mapgen": {F32: 2e-5, F16: 5e-3},
}
STATS_BAR = 1.5e-7      # fused InstanceNorm sums of the depthwise output against the sums of the output it stored


def _err(a, b):
    """max |a - b| / max |b|; absolute where b is exactly zero."""
    a, b = a.detach().double(), b.detach().double()
    scale = b.abs().max().item()
    return (a - b).abs().max().item() / (scale if scale > 0 else 1.0)


def _judge(kernel, tag, dtype, errs, special=False):
    print("MEDK_ERR %s %s %s %s" % (kernel, DT_ID[dtype], tag, json.dumps({k: float("%.3e" % v) for k, v in errs.items()})))
    bar = (SPECIAL_BARS if special else BARS)[kernel][dtype]
    bad = {k: v for k, v in errs.items() if not v < bar}
    assert not bad, (tag, bad, bar)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape, scale=1.0, dtype=F32):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


@pytest.fixture(scope="module")
def lib():
    import b200seg  # noqa: F401
    from b200seg import _lib
    assert _lib.load().b200seg_check_device() == 0, "not an H100"
    return _lib


# ============================================================================================ B-MHA (biattn.cu)
def _biattn_inputs(B, N, M, heads, dtype, seed, scale=1.5, peaked=False):
    g = _gen(seed)
    inner = 32 * heads
    fqv = _randn(g, B, N, 2 * inner, scale=scale)
    mqv = _randn(g, B, M, 2 * inner, scale=scale)
    if peaked:
        # map token j's column maximum on one voxel, in block (7 j) mod nblk: a different block, and merge partition
        # (block mod 4) cycling, for every token; that voxel's q is 3x the token's q, every other voxel's is small
        nblk = (N + 127) // 128
        fqv[..., :inner] *= 0.2
        for j in range(M):
            i = ((7 * j) % nblk) * 128 + (j * 13) % 128
            fqv[:, i, :inner] = 3.0 * mqv[:, j, :inner]
    dfo = _randn(g, B, N, inner)
    dmo = _randn(g, B, M, inner)
    return fqv.to(dtype), mqv.to(dtype), dfo.to(dtype), dmo.to(dtype)


def _biattn_reference(fqv, mqv, dfo, dmo, heads):
    """oracle.medformer_ops.bidirection_attention_core in float64 (tokens as an N x 1 x 1 volume)."""
    f = fqv.double().requires_grad_(True)
    m = mqv.double().requires_grad_(True)

    def vol(t):
        return t.permute(0, 2, 1)[..., None, None]
    fo, mo = mops.bidirection_attention_core(*vol(f).chunk(2, 1), *vol(m).chunk(2, 1), heads)
    fo, mo = fo[..., 0, 0].permute(0, 2, 1), mo[..., 0, 0].permute(0, 2, 1)
    torch.autograd.backward([fo, mo], [dfo.double(), dmo.double()])
    return fo.detach(), mo.detach(), f.grad, m.grad


def _biattn_check(tag, B, N, M, heads, dtype, seed, **kw):
    from b200seg.ops import BiAttnFn
    fqv, mqv, dfo, dmo = _biattn_inputs(B, N, M, heads, dtype, seed, **kw)
    f, m = fqv.clone().requires_grad_(True), mqv.clone().requires_grad_(True)
    fo, mo = BiAttnFn.apply(f, m, heads, 32)
    torch.autograd.backward([fo, mo], [dfo, dmo])
    rfo, rmo, rdf, rdm = _biattn_reference(fqv, mqv, dfo, dmo, heads)
    inner = 32 * heads
    errs = {"fo": _err(fo, rfo), "mo": _err(mo, rmo),
            "dfq": _err(f.grad[..., :inner], rdf[..., :inner]), "dfv": _err(f.grad[..., inner:], rdf[..., inner:]),
            "dmq": _err(m.grad[..., :inner], rdm[..., :inner]), "dmv": _err(m.grad[..., inner:], rdm[..., inner:])}
    _judge("biattn", tag, dtype, errs, special=kw.get("peaked", False) or kw.get("scale", 1.5) > 1.5)
    return errs


# M: 32-row build (1, 8, 27, 32) and 64-row build (33, 48, 64); N: one voxel, a block tail, exactly one block, one
# voxel into the second, and 3 / 4 / 5 blocks (merge partitions 1..3 empty, all four full, partition 0 twice with a
# ragged last block); heads cycle through 1 / 4 / 8 / 10 over the grid
BI_M = [1, 8, 27, 32, 33, 48, 64]
BI_N = [1, 127, 128, 129, 384, 512, 600]
BI_HEADS = [1, 4, 8, 10]
BI_ROWS = [(2, n, m, BI_HEADS[(a + b) % 4]) for a, m in enumerate(BI_M) for b, n in enumerate(BI_N)]
BI_ROWS += [(2, 1000, 27, h) for h in BI_HEADS] + [(2, 1000, 64, h) for h in BI_HEADS]
# the benchmark's levels (96^3 crop, map 3^3): down2 / up2, down3 / up1, down4
BI_BENCH = [(1, 55296, 27, 4), (1, 6912, 27, 8), (1, 864, 27, 10), (2, 55296, 27, 4), (2, 6912, 27, 8), (2, 864, 27, 10)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,N,M,heads", BI_ROWS, ids=["B%d-N%d-M%d-h%d" % r for r in BI_ROWS])
def test_biattn(B, N, M, heads, dtype):
    _biattn_check("B%d-N%d-M%d-h%d" % (B, N, M, heads), B, N, M, heads, dtype, seed=N + 100 * M + heads)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,N,M,heads", BI_BENCH, ids=["B%d-N%d-M%d-h%d" % r for r in BI_BENCH])
def test_biattn_bench_levels(B, N, M, heads, dtype):
    _biattn_check("bench-B%d-N%d-h%d" % (B, N, heads), B, N, M, heads, dtype, seed=7 + heads + B)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("row", ["peaked27", "peaked64", "large_logit"])
def test_biattn_special(row, dtype):
    """peaked: every map token's column maximum on one voxel, each in its own block and the merge partitions cycling,
    so the online rescale of both merges does the work; large_logit: q and k at 3x (|S| up to ~40)."""
    if row == "peaked27":
        _biattn_check(row, 2, 128 * 40, 27, 4, dtype, seed=11, peaked=True)
    elif row == "peaked64":
        _biattn_check(row, 2, 128 * 67, 64, 8, dtype, seed=12, peaked=True)
    else:
        _biattn_check(row, 2, 1000, 27, 8, dtype, seed=13, scale=4.5)


def _biattn_raw(lib, t, B, N, M, heads, dtype, ws):
    """b200seg_biattn_fwd / _bwd on caller-owned (ld, coff) buffers: t maps name -> (buffer, ld, coff)."""
    from b200seg.ops import _dt, _stream

    def p(name):
        return t[name][0].data_ptr()
    ld = {k: v[1] for k, v in t.items()}
    co = {k: v[2] for k, v in t.items()}
    colstat = torch.empty(B, heads, M, 2, device="cuda")
    lib.call("b200seg_biattn_fwd", p("fq"), ld["fq"], co["fq"], p("fv"), ld["fv"], co["fv"], p("mq"), co["mq"], p("mv"),
             co["mv"], ld["mq"], p("fo"), ld["fo"], co["fo"], p("mo"), ld["mo"], co["mo"], colstat.data_ptr(), ws.data_ptr(),
             B, N, M, heads, 32, 32 ** -0.5, _dt(t["fq"][0]), _stream())
    lib.call("b200seg_biattn_bwd", p("fq"), ld["fq"], co["fq"], p("fv"), ld["fv"], co["fv"], p("mq"), co["mq"], p("mv"),
             co["mv"], ld["mq"], p("mo"), ld["mo"], co["mo"], colstat.data_ptr(), p("dfo"), ld["dfo"], co["dfo"],
             p("dmo"), ld["dmo"], co["dmo"], p("dfq"), ld["dfq"], co["dfq"], p("dfv"), ld["dfv"], co["dfv"],
             p("dmq"), co["dmq"], p("dmv"), co["dmv"], ld["dmq"], ws.data_ptr(), B, N, M, heads, 32, 32 ** -0.5,
             _dt(t["fq"][0]), _stream())


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("N,M,heads", [(600, 27, 4), (129, 48, 8)])
def test_biattn_abi_sliced_operands(lib, N, M, heads, dtype):
    """Separate fq / fv / mq / mv / dfo / dmo and outputs, each at a non-zero channel offset inside a wider row, give
    the packed call's numbers bit for bit; outputs prefilled with NaN are fully written (their other channels are
    left alone); the workspace is exactly b200seg_biattn_workspace bytes (a canary just past it is untouched)."""
    from b200seg import ops
    B, inner = 2, 32 * heads
    fqv, mqv, dfo, dmo = _biattn_inputs(B, N, M, heads, dtype, seed=21)
    fo_p, mo_p, colstat = ops.biattn_fwd(fqv, mqv, heads)
    dfqv_p, dmqv_p = ops.biattn_bwd(fqv, mqv, mo_p, colstat, dfo, dmo, heads)
    t = {}

    def put(name, rows, src, coff, extra, nan=False):
        buf = torch.full((B, rows, coff + inner + extra), float("nan") if nan else 7.0, dtype=dtype, device="cuda")
        if src is not None:
            buf[..., coff:coff + inner] = src
        t[name] = (buf, buf.shape[-1], coff)
    put("fq", N, fqv[..., :inner], 8, 16)
    put("fv", N, fqv[..., inner:], 24, 40)
    put("dfo", N, dfo, 16, 8)
    put("fo", N, None, 40, 8, nan=True)
    put("dfq", N, None, 8, 24, nan=True)
    put("dfv", N, None, 32, 0, nan=True)
    # map-side operands share one row stride per call (m_ld for mq / mv, dm_ld for dmq / dmv)
    mbuf = torch.full((B, M, 2 * inner + 24), 7.0, dtype=dtype, device="cuda")
    mbuf[..., 8:8 + inner] = mqv[..., :inner]
    mbuf[..., 16 + inner:16 + 2 * inner] = mqv[..., inner:]
    t["mq"], t["mv"] = (mbuf, mbuf.shape[-1], 8), (mbuf, mbuf.shape[-1], 16 + inner)
    put("dmo", M, dmo, 24, 8)
    put("mo", M, None, 8, 8, nan=True)
    dm = torch.full((B, M, 2 * inner + 16), float("nan"), dtype=dtype, device="cuda")
    t["dmq"], t["dmv"] = (dm, dm.shape[-1], 16 + inner), (dm, dm.shape[-1], 0)
    nbytes = lib.load().b200seg_biattn_workspace(B, N, M, heads)
    wsbuf = torch.empty(nbytes // 4 + 64, dtype=torch.float32, device="cuda")
    canary = torch.randn(64, generator=_gen(22), device="cuda")
    wsbuf[nbytes // 4:] = canary
    _biattn_raw(lib, t, B, N, M, heads, dtype, wsbuf)
    torch.cuda.synchronize()
    assert torch.equal(wsbuf[nbytes // 4:], canary), "the kernels wrote past b200seg_biattn_workspace bytes"

    def cut(name):
        buf, _, coff = t[name]
        return buf[..., coff:coff + inner]
    for name, ref in (("fo", fo_p), ("mo", mo_p), ("dfq", dfqv_p[..., :inner]), ("dfv", dfqv_p[..., inner:]),
                      ("dmq", dmqv_p[..., :inner]), ("dmv", dmqv_p[..., inner:])):
        assert torch.equal(cut(name), ref), name
    # channels outside the written slices keep their NaN
    assert torch.isnan(t["fo"][0][..., :40]).all() and torch.isnan(t["dfq"][0][..., 8 + inner:]).all()
    assert torch.isnan(dm[..., inner:inner + 16]).all()


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_biattn_refusals(lib, dtype):
    """65 map tokens (over the 64-row build) and dim_head != 32 are errors, not truncated or misread attention."""
    from b200seg import ops
    f = torch.zeros(1, 4, 2 * 64, dtype=dtype, device="cuda")
    with pytest.raises(lib.B200SegError):
        ops.biattn_fwd(f, torch.zeros(1, 65, 2 * 64, dtype=dtype, device="cuda"), 2)
    with pytest.raises(lib.B200SegError):
        ops.biattn_fwd(f, torch.zeros(1, 8, 2 * 64, dtype=dtype, device="cuda"), 1, dim_head=64)
    f, m = torch.zeros(1, 4, 2 * 64, dtype=dtype, device="cuda"), torch.zeros(1, 65, 2 * 64, dtype=dtype, device="cuda")
    mo, colstat = torch.zeros(1, 65, 64, dtype=dtype, device="cuda"), torch.zeros(1, 2, 65, 2, device="cuda")
    with pytest.raises(lib.B200SegError):
        ops.biattn_bwd(f, m, mo, colstat, torch.zeros(1, 4, 64, dtype=dtype, device="cuda"), mo, 2)


# ============================================================================================ map generation
def _mapgen_check(tag, B, N, K, C, dtype, seed, pad=None, peaked=False):
    from b200seg.medformer_ops import MapGenFn
    g = _gen(seed)
    if pad is None:      # the module pads the fused projection to 16 channels; the backward takes <= 64 logit columns
        pad = (-(C + K)) % 16 if K + (-(C + K)) % 16 <= 64 else (-(C + K)) % 8
    fw = _randn(g, B, N, C + K + pad, scale=1.5)
    fw[..., C + K:] = 0
    if peaked:
        # code k's softmax over the voxels peaks on one voxel, in block (5 k) mod nblk
        nblk = (N + 127) // 128
        for k in range(K):
            fw[:, ((5 * k) % nblk) * 128 + (k * 11) % 128, C + k] = 12.0
    fw = fw.to(dtype)
    f64 = fw.double().requires_grad_(True)
    wm = F.softmax(f64[..., C:C + K], dim=1)                                   # softmax over the N voxels
    ref = torch.einsum("bnc,bnk->bkc", f64[..., :C], wm)
    gm = _randn(g, B, K, C).to(dtype)
    ref.backward(gm.double())
    x = fw.clone().requires_grad_(True)
    ms = (1, 1, K)
    smap = MapGenFn.apply(x, C, K, ms)
    smap.backward(gm.view(B, *ms, C))
    got = x.grad
    errs = {"map": _err(smap.view(B, K, C), ref), "dfeat": _err(got[..., :C], f64.grad[..., :C]),
            "dlogit": _err(got[..., C:C + K], f64.grad[..., C:C + K])}
    if pad:
        assert torch.count_nonzero(got[..., C + K:]) == 0, "logit padding columns must get zero gradient"
    _judge("mapgen", tag, dtype, errs, special=peaked)


MG_K = [1, 8, 27, 32, 33, 64]
MG_C = [8, 48, 56, 128, 320]        # 48 = one channel chunk, 56 = one chunk + 8, 320 = six chunks + 32
MG_N = [1, 127, 129, 1000]
MG_ROWS = [(2, MG_N[(a + b) % 4], k, c) for a, k in enumerate(MG_K) for b, c in enumerate(MG_C)]
MG_BENCH = [(1, 55296, 27, 128), (1, 6912, 27, 256), (1, 864, 27, 320)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,N,K,C", MG_ROWS + MG_BENCH, ids=["B%d-N%d-K%d-C%d" % r for r in MG_ROWS + MG_BENCH])
def test_mapgen(B, N, K, C, dtype):
    _mapgen_check("B%d-N%d-K%d-C%d" % (B, N, K, C), B, N, K, C, dtype, seed=N + K + C)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("row", ["peaked", "wide_pad"])
def test_mapgen_special(row, dtype):
    """peaked: each code's softmax maximum on one voxel of its own block; wide_pad: 27 codes padded to 64 logit
    channels (dw_pad beyond the 32-row build), whose gradient columns must be exactly zero."""
    if row == "peaked":
        _mapgen_check(row, 2, 128 * 40, 27, 128, dtype, seed=31, peaked=True)
    else:
        _mapgen_check(row, 2, 300, 27, 48, dtype, seed=32, pad=37)


def test_mapgen_bwd_refuses_unaligned_channels(lib):
    from b200seg.ops import _stream
    B, N, K, C = 1, 16, 8, 12
    fw = torch.zeros(B, N, C + K + 12, dtype=F16, device="cuda")
    smap = torch.zeros(B, K, C, dtype=F16, device="cuda")
    colstat = torch.ones(B, K, 2, device="cuda")
    ld = fw.shape[-1]
    with pytest.raises(lib.B200SegError):
        lib.call("b200seg_mapgen_bwd", fw.data_ptr(), ld, 0, fw.data_ptr(), ld, C, smap.data_ptr(), colstat.data_ptr(),
                 smap.data_ptr(), fw.data_ptr(), ld, 0, fw.data_ptr(), ld, C, ld - C, B, N, K, C, 1, _stream())


# ============================================================================================ MHSA
def _mhsa_check(tag, B, L, heads, dtype, seed, scale=1.0):
    from b200seg.medformer_ops import MHSAFn
    g = _gen(seed)
    inner = 32 * heads
    qkv = _randn(g, B, L, 3 * inner, scale=scale).to(dtype)
    dout = _randn(g, B, L, inner).to(dtype)
    x = qkv.clone().requires_grad_(True)
    out = MHSAFn.apply(x, heads, 32)
    out.backward(dout)
    q64 = qkv.double().requires_grad_(True)
    q, k, v = (t.reshape(B, L, heads, -1).permute(0, 2, 1, 3) for t in q64.chunk(3, dim=-1))
    att = F.softmax(torch.einsum("bhid,bhjd->bhij", q, k) * 32 ** -0.5, dim=-1)
    ref = torch.einsum("bhij,bhjd->bhid", att, v).permute(0, 2, 1, 3).reshape(B, L, -1)
    ref.backward(dout.double())
    errs = {"out": _err(out, ref)}
    for i, nm in enumerate(("dq", "dk", "dv")):
        errs[nm] = _err(x.grad[..., i * inner:(i + 1) * inner], q64.grad[..., i * inner:(i + 1) * inner])
    _judge("mhsa", tag, dtype, errs)


MH_L = [1, 27, 63, 64, 65, 81, 128, 192]
MH_ROWS = [(1 + (a + b) % 2, l, h) for a, l in enumerate(MH_L) for b, h in enumerate([1, 4, 8, 10])]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,L,heads", MH_ROWS, ids=["B%d-L%d-h%d" % r for r in MH_ROWS])
def test_mhsa(B, L, heads, dtype):
    _mhsa_check("B%d-L%d-h%d" % (B, L, heads), B, L, heads, dtype, seed=L * 16 + heads + B)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_mhsa_large_logit(dtype):
    _mhsa_check("large_logit", 2, 192, 4, dtype, seed=41, scale=3.0)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_mhsa_refuses_193_tokens(lib, dtype):
    from b200seg.medformer_ops import MHSAFn
    with pytest.raises(lib.B200SegError):
        MHSAFn.apply(torch.zeros(1, 193, 96, dtype=dtype, device="cuda"), 1, 32)


# ============================================================================================ LayerNorm, GELU
def _layernorm_check(lib, tag, R, C, dtype, seed, offset=0.0):
    """b200seg_layernorm_fwd / _bwd: y, dx, and d(gamma) / d(beta) added (+=) to prefilled buffers."""
    from b200seg.ops import _dt, _stream
    g = _gen(seed)
    x = (_randn(g, R, C) + offset).to(dtype)
    gamma, beta = 1 + 0.1 * _randn(g, C), 0.1 * _randn(g, C)
    dy = _randn(g, R, C).to(dtype)
    y, mr, dx = torch.empty_like(x), torch.empty(R, 2, device="cuda"), torch.empty_like(x)
    dg0, db0 = _randn(g, C), _randn(g, C)
    dg, db = dg0.clone(), db0.clone()
    lib.call("b200seg_layernorm_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mr.data_ptr(), R, C,
             1e-5, _dt(x), _stream())
    lib.call("b200seg_layernorm_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mr.data_ptr(), dx.data_ptr(),
             dg.data_ptr(), db.data_ptr(), R, C, _dt(x), _stream())
    x64, g64, b64 = (t.double().requires_grad_(True) for t in (x, gamma, beta))
    ref = F.layer_norm(x64, (C,), g64, b64, 1e-5)
    ref.backward(dy.double())
    errs = {"y": _err(y, ref), "dx": _err(dx, x64.grad), "dgamma": _err(dg - dg0, g64.grad), "dbeta": _err(db - db0, b64.grad)}
    _judge("layernorm", tag, dtype, errs)


LN_C = [32, 48, 96, 192, 320, 384, 768]
LN_R = [1, 5, 4224, 4225]          # 4224 = 132 * 8 blocks * 4 warps: beyond it a warp loops over several rows
LN_ROWS = [(r, c) for c in LN_C for r in LN_R] + [(262144, 48), (432, 768), (81, 320)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("R,C", LN_ROWS, ids=["R%d-C%d" % r for r in LN_ROWS])
def test_layernorm(lib, R, C, dtype):
    _layernorm_check(lib, "R%d-C%d" % (R, C), R, C, dtype, seed=R + C)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_layernorm_mean_far_above_std(lib, dtype):
    """|mean| = 300 x std: a one-pass E[x^2] - E[x]^2 variance would lose every digit."""
    _layernorm_check(lib, "offset300", 4225, 96, dtype, seed=51, offset=300.0)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("n", [1, 1001, 25920, 132 * 16 * 256 * 2 + 3])
def test_gelu(n, dtype):
    """odd n, the bench's 81 x 320 tokens, and n beyond one grid-stride pass; inputs spread over [-7, 7]."""
    from b200seg.medformer_ops import GeluFn
    g = _gen(n)
    x = (torch.rand(n, generator=g, device="cuda") * 14 - 7).to(dtype)
    dy = _randn(g, n).to(dtype)
    xg = x.clone().requires_grad_(True)
    y = GeluFn.apply(xg)
    y.backward(dy)
    x64 = x.double().requires_grad_(True)
    ref = F.gelu(x64)
    ref.backward(dy.double())
    _judge("gelu", "n%d" % n, dtype, {"y": _err(y, ref), "dx": _err(xg.grad, x64.grad)})


# ============================================================================================ SE gate + channel scale
def _se_check(tag, B, C, R, sp, dtype, seed):
    from b200seg.medformer_ops import SEScaleFn
    g = _gen(seed)
    x = (_randn(g, B, *sp, C) + 0.3).to(dtype)
    w1, b1 = _randn(g, R, C, 1, 1, 1, scale=C ** -0.5), _randn(g, R, scale=0.1)
    w2, b2 = _randn(g, C, R, 1, 1, 1, scale=R ** -0.5), _randn(g, C, scale=0.1)
    dy = _randn(g, B, *sp, C).to(dtype)
    xd = x.double().flatten(1, 3)
    st = torch.stack([xd.sum(1), (xd * xd).sum(1)], -1)
    ps = [t.clone().requires_grad_(True) for t in (w1, b1, w2, b2)]
    xg = x.clone().requires_grad_(True)
    y, _ = SEScaleFn.apply(xg, st, *ps)
    y.backward(dy)
    names = ("excitation.0.weight", "excitation.0.bias", "excitation.2.weight", "excitation.2.bias")
    sd64 = {k: t.double().requires_grad_(True) for k, t in zip(names, (w1, b1, w2, b2))}
    x64 = x.double().permute(0, 4, 1, 2, 3).requires_grad_(True)
    ref = omed.se_block(sd64, "", x64)
    ref.backward(dy.double().permute(0, 4, 1, 2, 3))
    errs = {"y": _err(y.permute(0, 4, 1, 2, 3), ref), "dx": _err(xg.grad.permute(0, 4, 1, 2, 3), x64.grad)}
    for k, p in zip(names, ps):
        errs["d" + k[11:].replace(".", "")] = _err(p.grad, sd64[k].grad)
    _judge("se", tag, dtype, errs)


# C = 1280 / 2048 put R > 256 (the second pass of se_gate_bwd's dz1 loop); 2048 gives the reduce one thread per
# channel octet (ncg >= 256); every V is not a multiple of the 256-thread blocks
SE_ROWS = [(b, c, max(1, c // 4), sp) for c, sp in ((8, (5, 6, 7)), (64, (9, 10, 11)), (512, (5, 6, 7)),
                                                     (1280, (3, 5, 7)), (2048, (3, 3, 5)))
           for b in (1, 2)]
SE_BENCH = [(1, 512, 128, (96, 24, 24)), (1, 1024, 256, (48, 12, 12)), (1, 1280, 320, (24, 6, 6))]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,C,R,sp", SE_ROWS + SE_BENCH, ids=["B%d-C%d-R%d-V%d" % (b, c, r, sp[0] * sp[1] * sp[2])
                                                              for b, c, r, sp in SE_ROWS + SE_BENCH])
def test_se_channel_scale(B, C, R, sp, dtype):
    _se_check("B%d-C%d-R%d-V%d" % (B, C, R, sp[0] * sp[1] * sp[2]), B, C, R, sp, dtype, seed=C + B)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,V,C", [(2, 1000, 4096), (1, 55296, 512), (2, 37, 8)])
def test_channel_scale_bwd_reduce(lib, B, V, C, dtype):
    """dgate += sum_vox dy * x beyond what the SE input statistics allow (C = 4096: 512 threads, one per channel octet):
    the gradient is added to a prefilled dgate, and two calls give the same bits."""
    from b200seg.ops import _dt, _stream
    g = _gen(C + V)
    dy, x = _randn(g, B, V, C).to(dtype), _randn(g, B, V, C).to(dtype)
    d0 = _randn(g, B, C)
    ws = torch.empty(lib.load().b200seg_channel_scale_bwd_workspace(B, V, C), dtype=torch.uint8, device="cuda")
    out = []
    for _ in range(2):
        dg = d0.clone()
        lib.call("b200seg_channel_scale_bwd_reduce", dy.data_ptr(), x.data_ptr(), dg.data_ptr(), ws.data_ptr(), B, V, C,
                 _dt(x), _stream())
        out.append(dg)
    assert torch.equal(out[0], out[1])
    ref = (dy.double() * x.double()).sum(1)
    _judge("se", "reduce-B%d-V%d-C%d" % (B, V, C), dtype, {"dgate": _err(out[0] - d0, ref)})


# ============================================================================================ space-to-depth, dwconv
# (B, Do, Ho, Wo, C, scale): the benchmark's PatchMerging calls (VEC = 8), then C not a multiple of 8 (VEC = 1)
S2D_BENCH = [(1, 96, 48, 48, 32, (1, 2, 2)), (1, 96, 24, 24, 64, (1, 2, 2)), (1, 48, 12, 12, 128, (2, 2, 2)),
             (1, 24, 6, 6, 256, (2, 2, 2))]
S2D_ROWS = S2D_BENCH + [(2, 5, 6, 7, 1, (2, 2, 2)), (2, 4, 6, 5, 12, (1, 2, 2)), (1, 3, 4, 5, 3, (2, 1, 2))]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,Do,Ho,Wo,C,s", S2D_ROWS, ids=["B%d-%dx%dx%d-C%d-s%d%d%d" % (*r[:5], *r[5]) for r in S2D_ROWS])
def test_space_to_depth(lib, B, Do, Ho, Wo, C, s, dtype):
    """y[..., q*C + c] = x[b, d*sd+i, h*sh+j, w*sw+k, c] with q = (i*sh + j)*sw + k, and its scatter back: bit-exact."""
    from b200seg.ops import _dt, _stream
    sd, sh, sw = s
    x = _randn(_gen(C + Do), B, Do * sd, Ho * sh, Wo * sw, C).to(dtype)
    y = torch.full((B, Do, Ho, Wo, C * sd * sh * sw), float("nan"), dtype=dtype, device="cuda")
    lib.call("b200seg_space_to_depth", x.data_ptr(), y.data_ptr(), B, Do, Ho, Wo, C, sd, sh, sw, 0, _dt(x), _stream())
    ref = torch.cat([x[:, i::sd, j::sh, k::sw, :] for i in range(sd) for j in range(sh) for k in range(sw)], -1)
    assert torch.equal(y, ref)
    back = torch.full_like(x, float("nan"))
    lib.call("b200seg_space_to_depth", back.data_ptr(), y.data_ptr(), B, Do, Ho, Wo, C, sd, sh, sw, 1, _dt(x), _stream())
    assert torch.equal(back, x)


# (B, D, H, W, C, k): every depthwise call of the benchmark (PatchMerging reductions, feat_qv / feat_out, MBConv) --
# C = 320 and 576 run channel slices of 80 and 96 (pick_chunk < 128) -- and two small edge rows
DW_BENCH = [(1, 96, 48, 48, 128, (1, 3, 3)), (1, 96, 24, 24, 256, (3, 3, 3)), (1, 96, 24, 24, 128, (3, 3, 3)),
            (1, 96, 24, 24, 512, (3, 3, 3)), (1, 96, 24, 24, 384, (3, 3, 3)), (1, 48, 12, 12, 1024, (3, 3, 3)),
            (1, 48, 12, 12, 256, (3, 3, 3)), (1, 48, 12, 12, 576, (3, 3, 3)), (1, 24, 6, 6, 2048, (3, 3, 3)),
            (1, 24, 6, 6, 320, (3, 3, 3)), (1, 24, 6, 6, 1280, (3, 3, 3))]
DW_ROWS = DW_BENCH + [(2, 5, 7, 9, 40, (1, 3, 3)), (2, 3, 4, 5, 8, (3, 3, 3)), (2, 1, 6, 11, 48, (3, 3, 3))]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,D,H,W,C,k", DW_ROWS, ids=["B%d-%dx%dx%d-C%d-k%d%d%d" % (*r[:5], *r[5]) for r in DW_ROWS])
def test_dwconv(B, D, H, W, C, k, dtype):
    """forward on relu(IN(x)) from the producer's sums, with the fused sums of its output; the data gradient (the
    flipped forward); the weight gradient -- each against float64 on the kernel's rounded operands."""
    from b200seg import ops
    g = _gen(C + D)
    eps = 1e-4
    x = (_randn(g, B, D, H, W, C, scale=1.5) + 0.2).to(dtype)
    w = _randn(g, C, 1, *k, scale=0.3)
    dy = _randn(g, B, D, H, W, C).to(dtype)
    xd = x.double().flatten(1, 3)
    st = torch.stack([xd.sum(1), (xd * xd).sum(1)], -1)
    y, yst = ops.dwconv3d(x, w, k, x_stats=st, act=ops.ACT_RELU, want_stats=True, eps=eps, cmajor=True)
    dx, _ = ops.dwconv3d(dy, w, k, flip=True, cmajor=True)
    dw = ops.dwconv3d_wgrad(x, dy, k, x_stats=st, act=ops.ACT_RELU, eps=eps, cmajor=True)
    x64 = x.double().permute(0, 4, 1, 2, 3)
    a = F.relu(F.instance_norm(x64, eps=eps)).to(dtype).double().requires_grad_(True)   # the kernel rounds a to T
    w64 = w.double().requires_grad_(True)
    ref = mops.depthwise_conv3d(a, w64)
    ref.backward(dy.double().permute(0, 4, 1, 2, 3))
    yd = y.double().flatten(1, 3)
    errs = {"y": _err(y.permute(0, 4, 1, 2, 3), ref), "dx": _err(dx.permute(0, 4, 1, 2, 3), a.grad),
            "dw": _err(dw, w64.grad)}
    stat_err = _err(yst, torch.stack([yd.sum(1), (yd * yd).sum(1)], -1))
    print("MEDK_ERR dwconv_stats %s B%d-C%d %.3e" % (DT_ID[dtype], B, C, stat_err))
    assert stat_err < STATS_BAR
    _judge("dwconv", "B%d-%dx%dx%d-C%d" % (B, D, H, W, C), dtype, errs)


# ============================================================================================ the benchmark's shapes
BCV = dict(map_size=[3, 3, 3], conv_num=[2, 0, 0, 0, 0, 0, 2, 2], trans_num=[0, 2, 4, 6, 4, 2, 0, 0],
           num_heads=[1, 4, 8, 10, 8, 4, 1, 1], fusion_depth=2, fusion_dim=320, fusion_heads=10,
           kernel_size=[[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
           scale=[[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2]], aux_loss=True)
AUX_WEIGHT = [0.5, 0.5]


def _bcv_args():
    c = dict(BCV)
    return types.SimpleNamespace(dimension="3d", model="medformer", in_chan=1, classes=14, base_chan=32,
                                 conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0, proj_type="depthwise",
                                 norm="in", act="relu", down_scale=c.pop("scale"), **c)


def _bcv_state(net):
    """Seeded weights for the benchmarked MedFormer that keep it out of the chaotic regime, so that fp16 rounding
    moves its logits and gradients by ~1e-2 (stock autocast of the oracle: logits 4.4e-3, gradient global L2 1.3e-2)
    rather than by 50-100%.  make_state_dict draws every tensor at 1/sqrt(fan_in), which gives 1-D tensors (biases)
    unit scale; at that scale the 55 296-voxel softmaxes of map generation and B-MHA are so peaked, and the 18
    undamped residual branches so amplifying, that stock autocast differs from fp32 by 0.48 in the logits.  So: 1-D
    tensors within +-0.1 (norm.weight 1 +- 0.1), the map-code logits (semantic_proj) and the attention q / v
    projections scaled down, and the last projection of every residual branch at 0.2 (a near-identity block)."""
    sd = ounet.make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=7)
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


def _table_keys():
    """the shape keys the tables above run, per entry point family"""
    return {
        "biattn": {(b, n, m, h) for b, n, m, h in BI_ROWS + BI_BENCH},
        "mapgen": {(b, n, k, c) for b, n, k, c in MG_ROWS + MG_BENCH},
        "mhsa": {(b, l, h) for b, l, h in MH_ROWS},
        "layernorm": {(r, c) for r, c in LN_ROWS},
        "gelu": {1, 1001, 25920, 132 * 16 * 256 * 2 + 3},
        "se_gate": {(b, c, r) for b, c, r, _ in SE_ROWS + SE_BENCH},
        "channel_scale": {(b, sp[0] * sp[1] * sp[2], c) for b, c, _, sp in SE_ROWS + SE_BENCH},
        "dwconv3d": {(b, d, h, w, c, *k) for b, d, h, w, c, k in DW_ROWS},
        "space_to_depth": {(b, do, ho, wo, c, *s) for b, do, ho, wo, c, s in S2D_ROWS},
    }


def _shape_key(name, args):
    """entry point -> (family, shape key) from the raw C-ABI arguments (include/b200seg.h)."""
    n = name[len("b200seg_"):]
    if n.startswith("biattn_"):
        return "biattn", tuple(args[-8:-4])
    if n.startswith("mapgen_"):
        return "mapgen", tuple(args[-6:-2])
    if n == "mhsa":
        return "mhsa", tuple(args[4:7])
    if n == "layernorm_fwd":
        return "layernorm", tuple(args[5:7])
    if n == "layernorm_bwd":
        return "layernorm", tuple(args[7:9])
    if n == "gelu":
        return "gelu", args[3]
    if n.startswith("se_gate_"):
        return "se_gate", (tuple(args[9:12]) if n == "se_gate_fwd" else tuple(args[-4:-1]))
    if n.startswith("channel_scale_") and not n.endswith("workspace"):
        return "channel_scale", tuple(args[-5:-2])
    if n.startswith("dwconv3d_"):
        return "dwconv3d", tuple(args[-10:-2])
    if n == "space_to_depth":
        return "space_to_depth", tuple(args[2:10])
    return None, None


def test_bench_call_shapes_are_in_the_tables(monkeypatch):
    """One AMP forward / backward of the benchmarked MedFormer (medformer_bcv_96: 96^3, 14 classes, map 3^3) with every
    call into the library recorded: each B-MHA, map generation, MHSA, LayerNorm, GELU, SE, channel-scale, depthwise and
    space-to-depth shape it uses is a row of the tables above."""
    import b200seg
    from b200seg import medformer_ops, ops
    seen = {}

    def recorder(real):
        def call(name, *args):
            fam, key = _shape_key(name, args)
            if fam is not None:
                seen.setdefault(fam, set()).add(key)
            return real(name, *args)
        return call
    for mod in (ops, medformer_ops):
        monkeypatch.setattr(mod, "call", recorder(mod.call))
    net = b200seg.get_model(_bcv_args())
    net.load_state_dict(_bcv_state(net))
    net = net.cuda()
    img, lab = make_volume(1, 96, 96, 96, 14, seed=2026)
    with torch.autocast("cuda", dtype=torch.float16):
        res = net(img.cuda())
        loss = sum(wt * b200seg.DiceCELoss(weight=torch.tensor([0.5] + [1.0] * 13))(r, lab.cuda())
                   for wt, r in zip(AUX_WEIGHT, res))
    (loss * 1024.0).backward()
    torch.cuda.synchronize()
    tables = _table_keys()
    print("MedFormer bcv 96 call shapes: %s" % {k: sorted(v) for k, v in seen.items()})
    assert set(seen) == set(tables), set(seen) ^ set(tables)
    for fam, keys in seen.items():
        assert keys <= tables[fam], (fam, sorted(keys - tables[fam]))


def _bcv_setup():
    import b200seg
    net = b200seg.get_model(_bcv_args())
    sd = _bcv_state(net)
    img, lab = make_volume(1, 96, 96, 96, 14, seed=2026)
    return sd, img.cuda(), lab.cuda(), torch.tensor([0.5] + [1.0] * 13)


def test_fullsize_amp_step():
    """get_model's MedFormer as bench.py times it (medformer_bcv_96: 96^3, 14 classes, aux head, AMP): one forward /
    backward against the fp32 oracle, with stock torch autocast of the same oracle as the fp16 noise floor.  The bars
    are those of the SwinUNETR and UNETR full-size steps; a zeroed gradient (global L2 1.0) or zeroed logits fail."""
    import b200seg
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        sd, img, lab, w = _bcv_setup()

        def oracle(autocast, S):
            s = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                lo = omed.medformer_forward(s, img, BCV)
                loss = olosses.total_loss(lo, lab, w.cuda(), AUX_WEIGHT)
            (loss * S).backward()
            return ([t.detach().double().cpu() for t in lo], loss.item(),
                    {k: (v.grad / S).double().cpu() for k, v in s.items()})
        l32, loss32, g32 = oracle(False, 1.0)
        l_st, loss_st, g_st = oracle(True, 1024.0)
        torch.cuda.empty_cache()

        net = b200seg.get_model(_bcv_args())
        net.load_state_dict(sd)
        net = net.cuda()
        S = 1024.0
        with torch.autocast("cuda", dtype=torch.float16):
            res = net(img)
            crit = b200seg.DiceCELoss(weight=w)
            loss = sum(wt * crit(r, lab) for wt, r in zip(AUX_WEIGHT, res))
        (loss * S).backward()
        lg = [r.detach().double().cpu() for r in res]
        ours = {k: (p.grad / S).double().cpu() for k, p in net.named_parameters()}
        assert set(ours) == set(g32)
        assert all(torch.isfinite(v).all() for v in ours.values())
        e = max(rel_err(a, b) for a, b in zip(lg, l32))
        e_st = max(rel_err(a, b) for a, b in zip(l_st, l32))
        l2, l2_st = global_l2(ours, g32), global_l2(g_st, g32)
        agree = (lg[0].argmax(1) == l32[0].argmax(1)).float().mean().item()
        agree_st = (l_st[0].argmax(1) == l32[0].argmax(1)).float().mean().item()
        print("medformer bcv 96 AMP: logits rel err vs fp32 oracle %.2e (stock autocast %.2e); loss %.5f (oracle %.5f, "
              "stock autocast %.5f); grads global-L2 %.2e (stock autocast %.2e); label agreement %.5f (stock autocast %.5f)"
              % (e, e_st, loss.item(), loss32, loss_st, l2, l2_st, agree, agree_st))
        assert e < max(5e-2, 3 * e_st)
        assert abs(loss.item() - loss32) < 2e-2
        assert l2 < max(0.1, 3 * l2_st)
        assert agree > 0.97
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def test_fullsize_trainstep_reproducible():
    """Two identical TrainSteps of the benchmarked MedFormer from the same state give the same loss and bit-identical
    parameters and EMA, outside the parameters whose gradients are summed with float atomics (DESIGN §4a)."""
    import b200seg
    from b200seg.train import TrainStep
    sd, img, lab, w = _bcv_setup()
    args = _bcv_args()

    def one_step():
        n = b200seg.get_model(args)
        n.load_state_dict(sd)
        n = n.cuda()
        ema = b200seg.get_model(args)
        ema.load_state_dict(sd)
        ema = ema.cuda()
        step = TrainStep(n, ema, ce_weight=w, amp=True, aux_weight=AUX_WEIGHT)
        step.fused.scale.fill_(1024.0)      # a first step at GradScaler's 65536 may overflow in fp16 and be skipped
        lv = step(img, lab)
        torch.cuda.synchronize()
        return (lv.item(), [(k, p.detach().cpu()) for k, p in n.named_parameters()],
                [p.detach().cpu() for p in ema.parameters()])
    la, pa, ea = one_step()
    torch.cuda.empty_cache()
    lb, pb, eb = one_step()
    moved = sum(1 for k, p in pa if not torch.equal(p, sd[k]))
    differ = [k for (k, x), (_, y), u, v in zip(pa, pb, ea, eb) if not (torch.equal(x, y) and torch.equal(u, v))]
    print("medformer bcv 96 TrainStep: loss %.6f / %.6f, %d of %d parameter tensors updated; differing between the "
          "two runs (%d): %s" % (la, lb, moved, len(pa), len(differ), differ))
    assert la == lb
    assert moved > len(pa) // 2

    def atomic(k):
        # dwconv_wgrad_kernel adds its per-block depthwise weight-gradient partials with float atomics
        if k.endswith("depthwise.weight") or k.endswith("depthwise.conv.weight"):
            return True
        # LayerNormFn's backward (b200seg_layernorm_bwd) sums d(gamma) / d(beta) with float atomics
        return ".norm" in k and k.split(".")[-1] in ("weight", "bias")
    assert all(atomic(k) for k in differ), [k for k in differ if not atomic(k)]
