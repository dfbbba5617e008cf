"""GPU: the convolution and InstanceNorm kernels on channel-sliced operands, and the tensor-core routing limits.

Every activation operand of the C ABI is a (ld, coff) slice: channels coff .. coff+C of a buffer with ld channels per
voxel.  The ResUNet block reads and writes such slices on every step (conv1 + shortcut as one GEMM of width 2*Cout).
Here each sliced operand is built as a wider buffer whose other channels hold finite poison, each sliced output as a
wider buffer whose other channels hold a sentinel that must survive bit for bit.  Every call is checked twice:
  * against the same call on dense tensors: bit-identical wherever the slice takes the same kernel path as the dense
    call (the staging path is chosen from the shape, not from ld / coff);
  * against PyTorch in fp64 on the same fp16-rounded inputs: 3e-3 to 4e-3 in fp16, 1e-4 in fp32.

Which tensor-core staging path each forward row reaches (host-side selection in conv_tc.cu), and which weight-gradient
loader (wgrad_tc.cu fill_params):
  forward  raw TMA: "tma_raw", "tma_raw_dgrad"; TMA + in-place transform: "tma_xform_32", "tma_xform_64";
           cp.async 3 stages: "cpasync3_96", "cpasync3_128"; cp.async 1 stage: "cpasync1_b64"
  wgrad    wg_loader<3>: Cin 32; wg_loader<2>: Cin 128; wg_loader<1>: Cin 192
"""
import pytest
import torch
import torch.nn.functional as F

from util import assert_untouched, global_l2, rel_err, sentinel, wide

pytestmark = pytest.mark.gpu

EPS = 1e-4
TOL32, TOL16 = 1e-4, 4e-3


@pytest.fixture(scope="module")
def lib():
    import b200seg
    from b200seg import _lib, ops  # noqa: F401
    assert _lib.load().b200seg_check_device() == 0, "not an H100"
    return b200seg


# ----------------------------------------------------------------------------- operands
def randh(*shape, dtype=torch.float16, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def stats64(t):
    """[B, D, H, W, C] -> InstanceNorm sums [B, C, 2] (fp64) of the stored values."""
    d = t.double().flatten(1, 3)
    return torch.stack([d.sum(1), (d * d).sum(1)], -1).contiguous()


def nc(t):
    return t.detach().double().cpu().permute(0, 4, 1, 2, 3)


def xhat64(t, st):
    """(x - mean) * rstd in fp64, NCDHW on the CPU, from the sums the kernels are given"""
    n = t[0, ..., 0].numel()
    st = st.double().cpu()
    m = st[..., 0] / n
    r = 1.0 / torch.sqrt((st[..., 1] / n - m * m).clamp_min(0) + EPS)
    return (nc(t) - m[:, :, None, None, None]) * r[:, :, None, None, None]


def act64(h, act):
    return h if act == 0 else (h.clamp_min(0) if act == 1 else torch.where(h > 0, h, 0.01 * h))


def dact64(h, act):
    one = torch.ones_like(h)
    return one if act == 0 else torch.where(h > 0, one, torch.zeros_like(h) if act == 1 else 0.01 * one)


def rnd(t, dtype):
    return t.to(dtype).double()


def same(a, b, exact, tol=1e-6):
    if exact:
        assert torch.equal(a, b)
    else:
        assert rel_err(a.float(), b.float()) < tol


def _p(t):
    return None if t is None else t.data_ptr()


def conv_raw(lib, x, x_coff, x_st, act, wp, y, y_coff, y_st, Cin, Cout, k, algo,
             res=None, r_coff=0, gx=None, gx_coff=0, g_st=None, bias=None):
    """b200seg_conv3d_fwd with every (ld, coff) taken from the buffers: ld = the buffer's channel count."""
    ops = lib.ops
    B, D, H, W, _ = y.shape
    lib._lib.call("b200seg_conv3d_fwd", x.data_ptr(), x.shape[-1], x_coff, _p(x_st), EPS, act, wp.data_ptr(), _p(bias),
                  _p(res), 0 if res is None else res.shape[-1], r_coff, y.data_ptr(), y.shape[-1], y_coff, _p(y_st),
                  _p(gx), 0 if gx is None else gx.shape[-1], gx_coff, _p(g_st), EPS, ops.ACT_RELU if gx is not None else 0,
                  B, D, H, W, Cin, Cout, *k, ops._dt(x), algo, ops._stream())


def zstats(B, C, n=2):
    return torch.zeros(B, C, n, dtype=torch.float64, device="cuda")


# ----------------------------------------------------------------------------- tensor-core forward
FWD_ROWS = {
    # name: (Cin, Cout, k, (B, D, H, W), mode); H and W are ragged against the 16 x 8 output tile
    "tma_raw": (16, 16, (1, 1, 1), (1, 2, 20, 12), "plain"),
    "tma_raw_dgrad": (64, 32, (3, 3, 3), (2, 3, 20, 12), "dgrad"),
    "tma_xform_32": (32, 64, (3, 3, 3), (2, 3, 20, 12), "normres"),
    "tma_xform_64": (64, 64, (1, 3, 3), (1, 2, 36, 20), "norm"),
    "cpasync3_96": (96, 64, (1, 3, 3), (1, 2, 36, 20), "normres"),
    "cpasync3_128": (128, 128, (3, 3, 3), (1, 2, 20, 12), "norm"),
    "cpasync1_b64": (64, 32, (3, 3, 3), (64, 1, 18, 10), "norm"),     # B*Cin tables leave room for 3 A stages only
}
# (x_ld, x_coff); the widest layout also writes its output into a slice (y_ld = Cout + 16, y_coff = 8)
X_LAYOUTS = {"ld+16": (16, 0), "ld+16_coff16": (16, 16), "ldx2": (None, 0), "ldx2_coff16": (None, 16)}


@pytest.mark.parametrize("layout", list(X_LAYOUTS))
@pytest.mark.parametrize("row", list(FWD_ROWS))
def test_tc_fwd_sliced_operands(lib, row, layout):
    ops = lib.ops
    Cin, Cout, k, (B, D, H, W), mode = FWD_ROWS[row]
    extra, x_coff = X_LAYOUTS[layout]
    x_ld = Cin + extra if extra else 2 * Cin
    out_slice = layout == "ldx2_coff16"
    taps = k[0] * k[1] * k[2]
    x = randh(B, D, H, W, Cin, seed=1)
    w = (torch.randn(Cout, Cin, *k, generator=torch.Generator().manual_seed(2)) / (Cin * taps) ** 0.5).cuda()
    assert ops.conv_algo(Cin, Cout, k, torch.float16, B) == ops.ALGO_TC
    wp = ops.pack_weight(w, torch.float16, layout=ops.ALGO_TC)
    norm = mode in ("norm", "normres")
    xst = stats64(x) if norm else None
    act = ops.ACT_RELU if norm else ops.ACT_NONE
    res = randh(B, D, H, W, Cout, seed=3) if mode == "normres" else None
    gx = randh(B, D, H, W, Cout, seed=4) if mode == "dgrad" else None
    gst = stats64(gx) if gx is not None else None

    yd, sd = torch.empty(B, D, H, W, Cout, dtype=torch.float16, device="cuda"), zstats(B, Cout)
    conv_raw(lib, x, 0, xst, act, wp, yd, 0, sd, Cin, Cout, k, ops.ALGO_TC, res=res, gx=gx, g_st=gst)
    y_ld, y_coff = (Cout + 16, 8) if out_slice else (Cout, 0)
    ys, ss = sentinel((B, D, H, W), y_ld, torch.float16), zstats(B, Cout)
    conv_raw(lib, wide(x, x_ld, x_coff), x_coff, xst, act, wp, ys, y_coff, ss, Cin, Cout, k, ops.ALGO_TC,
             res=None if res is None else wide(res, 2 * Cout, Cout), r_coff=Cout,       # the BasicBlock shortcut half
             gx=None if gx is None else wide(gx, 2 * Cout, 0), g_st=gst)               # conv2's dgrad reads ts
    torch.cuda.synchronize()
    assert torch.equal(ys[..., y_coff:y_coff + Cout], yd)
    assert_untouched(ys, y_coff, Cout)
    assert rel_err(ss, sd) < 1e-12

    wd = w.half().double().cpu()
    pad = [i // 2 for i in k]
    if mode == "dgrad":
        h = xhat64(gx, gst)
        ref = F.conv3d(nc(x), wd, padding=pad) * dact64(h, ops.ACT_RELU)
        y64 = nc(yd)
        sref = torch.stack([y64.sum((2, 3, 4)), (y64 * h).sum((2, 3, 4))], -1)
        assert rel_err(sd, sref) < 1e-4
    else:
        a = rnd(act64(xhat64(x, xst), act), torch.float16) if norm else nc(x)
        ref = F.conv3d(a, wd, padding=pad)
        if res is not None:
            ref = rnd(ref, torch.float16) + nc(res)
        assert rel_err(sd, stats64(yd)) < 1e-5          # the sums describe what was stored
    assert rel_err(nc(yd), ref) < 4e-3


# ----------------------------------------------------------------------------- tensor-core weight gradient
WG_ROWS = {
    "wg_loader3": (32, 32, (3, 3, 3), (1, 3, 20, 12)),
    "wg_loader2": (128, 128, (3, 3, 3), (1, 2, 20, 12)),
    "wg_loader1": (192, 256, (3, 3, 3), (1, 2, 16, 16)),
}
# (x_ld extra or None = 2*Cin, x_coff, dy_ld extra or None = 2*Cout, dy_coff)
WG_LAYOUTS = {"x_ld+16_coff16__dy_ldx2_coffC": (16, 16, None, "C"), "x_ldx2__dy_ld+16_coff16": (None, 0, 16, 16)}


def _wg_slices(Cin, Cout, lay):
    xe, x_coff, de, dy_coff = lay
    x_ld = Cin + xe if xe else 2 * Cin
    dy_ld = Cout + de if de else 2 * Cout
    return x_ld, x_coff, dy_ld, Cout if dy_coff == "C" else dy_coff


def _wgrad64(x, xst, act, dy, k, Cout, bias=False):
    a = rnd(act64(xhat64(x, xst), act), torch.float16) if xst is not None else nc(x)
    w = torch.zeros(Cout, a.shape[1], *k, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(Cout, dtype=torch.float64, requires_grad=True) if bias else None
    F.conv3d(a, w, b, padding=[i // 2 for i in k]).backward(nc(dy))
    return w.grad, None if b is None else b.grad


@pytest.mark.parametrize("layout", list(WG_LAYOUTS))
@pytest.mark.parametrize("row", list(WG_ROWS))
def test_tc_wgrad_sliced_operands(lib, row, layout):
    ops = lib.ops
    Cin, Cout, k, (B, D, H, W) = WG_ROWS[row]
    x_ld, x_coff, dy_ld, dy_coff = _wg_slices(Cin, Cout, WG_LAYOUTS[layout])
    x = randh(B, D, H, W, Cin, seed=5)
    dy = randh(B, D, H, W, Cout, seed=6)
    xst = stats64(x)
    dwd, _ = ops.conv3d_wgrad(x, 0, Cin, xst, ops.ACT_RELU, dy, 0, Cout, k, algo=ops.ALGO_TC)
    dws, _ = ops.conv3d_wgrad(wide(x, x_ld, x_coff), x_coff, Cin, xst, ops.ACT_RELU, wide(dy, dy_ld, dy_coff), dy_coff,
                              Cout, k, algo=ops.ALGO_TC)
    torch.cuda.synchronize()
    assert torch.equal(dws, dwd)              # split-K partials are summed in a fixed order
    ref, _ = _wgrad64(x, xst, ops.ACT_RELU, dy, k, Cout)
    assert rel_err(dwd, ref) < 3e-3


@pytest.mark.parametrize("Cin,Cout,k,shape", [(48, 144, (1, 1, 1), (1, 8, 16, 16)), (32, 24, (3, 3, 3), (1, 3, 20, 12))])
def test_tc_wgrad_with_bias_sliced_operands(lib, Cin, Cout, k, shape):
    """ALGO_AUTO with a bias gradient: the column-sum pass (bias_grad_kernel, its own dy_ld / dy_coff) + the tensor cores."""
    ops = lib.ops
    B, D, H, W = shape
    x = randh(B, D, H, W, Cin, seed=7)
    dy = randh(B, D, H, W, Cout, seed=8)
    dwd, dbd = ops.conv3d_wgrad(x, 0, Cin, None, ops.ACT_NONE, dy, 0, Cout, k, want_bias=True)
    dws, dbs = ops.conv3d_wgrad(wide(x, Cin + 16, 16), 16, Cin, None, ops.ACT_NONE, wide(dy, 2 * Cout, Cout), Cout,
                                Cout, k, want_bias=True)
    torch.cuda.synchronize()
    assert torch.equal(dws, dwd) and torch.equal(dbs, dbd)
    wref, bref = _wgrad64(x, None, 0, dy, k, Cout, bias=True)
    assert rel_err(dwd, wref) < 3e-3 and rel_err(dbd, bref) < 1e-3


# ----------------------------------------------------------------------------- CUDA-core and special kernels
DIRECT_ROWS = {
    # (Cin, Cout, k, (B, D, H, W), x_ld, x_coff): tensor-core shapes, but slices the tensor cores refuse
    "coff4": (16, 32, (3, 3, 3), (2, 3, 9, 11), 20, 4),
    "ld_odd": (32, 16, (1, 3, 3), (2, 3, 9, 11), 37, 3),
}
DTYPES = {"fp32": (torch.float32, TOL32), "fp16": (torch.float16, TOL16)}


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("row", list(DIRECT_ROWS))
def test_direct_fwd_unaligned_slices(lib, row, dt):
    """ALGO_DIRECT forward with InstanceNorm+ReLU, a residual slice, fused sums and an output slice."""
    ops = lib.ops
    dtype, tol = DTYPES[dt]
    Cin, Cout, k, (B, D, H, W), x_ld, x_coff = DIRECT_ROWS[row]
    x = randh(B, D, H, W, Cin, dtype=dtype, seed=9)
    res = randh(B, D, H, W, Cout, dtype=dtype, seed=10)
    w = (torch.randn(Cout, Cin, *k, generator=torch.Generator().manual_seed(11)) * 0.2).cuda()
    wp = ops.pack_weight(w, dtype)
    xst = stats64(x)
    xs, rs = wide(x, x_ld, x_coff), wide(res, Cout + 5, 2)
    ys, ss = sentinel((B, D, H, W), Cout + 3, dtype), zstats(B, Cout)
    if dtype == torch.float16:        # the tensor cores refuse the slice before launching anything
        with pytest.raises(lib._lib.B200SegError):
            conv_raw(lib, xs, x_coff, xst, ops.ACT_RELU, wp, ys, 1, ss, Cin, Cout, k, ops.ALGO_TC, res=rs, r_coff=2)
    conv_raw(lib, xs, x_coff, xst, ops.ACT_RELU, wp, ys, 1, ss, Cin, Cout, k, ops.ALGO_DIRECT, res=rs, r_coff=2)
    yd, sd = torch.empty(B, D, H, W, Cout, dtype=dtype, device="cuda"), zstats(B, Cout)
    conv_raw(lib, x, 0, xst, ops.ACT_RELU, wp, yd, 0, sd, Cin, Cout, k, ops.ALGO_DIRECT, res=res)
    torch.cuda.synchronize()
    assert_untouched(ys, 1, Cout)
    y = ys[..., 1:1 + Cout]
    # the dense call loads 8 channels at a time, the slice one: a different summation order
    same(y, yd, exact=False, tol=1e-5 if dtype == torch.float32 else 2e-3)
    a = rnd(act64(xhat64(x, xst), ops.ACT_RELU), dtype)
    ref = rnd(F.conv3d(a, rnd(w.cpu(), dtype), padding=[i // 2 for i in k]), dtype) + nc(res)
    assert rel_err(nc(y), ref) < tol
    assert rel_err(ss, stats64(y)) < 1e-5


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("row", list(DIRECT_ROWS))
def test_direct_wgrad_unaligned_slices(lib, row, dt):
    ops = lib.ops
    dtype, tol = DTYPES[dt]
    Cin, Cout, k, (B, D, H, W), x_ld, x_coff = DIRECT_ROWS[row]
    x = randh(B, D, H, W, Cin, dtype=dtype, seed=12)
    dy = randh(B, D, H, W, Cout, dtype=dtype, seed=13)
    xst = stats64(x)
    dws, _ = ops.conv3d_wgrad(wide(x, x_ld, x_coff), x_coff, Cin, xst, ops.ACT_RELU, wide(dy, Cout + 5, 3), 3, Cout, k,
                              algo=ops.ALGO_AUTO)
    dwd, _ = ops.conv3d_wgrad(x, 0, Cin, xst, ops.ACT_RELU, dy, 0, Cout, k, algo=ops.ALGO_DIRECT)
    torch.cuda.synchronize()
    assert rel_err(dws, dwd) < 1e-5           # fp32 atomics: the order of the additions varies
    a = rnd(act64(xhat64(x, xst), ops.ACT_RELU), dtype)
    w = torch.zeros(Cout, Cin, *k, dtype=torch.float64, requires_grad=True)
    F.conv3d(a, w, padding=[i // 2 for i in k]).backward(nc(dy))
    assert rel_err(dws, w.grad) < max(tol, 2e-3 if dtype == torch.float16 else tol)


# the 1x1x1 few-class head (small_conv.cu): (x_ld, x_coff, y_ld, y_coff, takes the vector kernel)
HEAD_FWD = {"x4_vector": (36, 4, 8, 4, True), "x2_scalar": (34, 2, 6, 2, False)}


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(HEAD_FWD))
def test_head_fwd_sliced(lib, layout, dt):
    ops = lib.ops
    dtype, _ = DTYPES[dt]
    tol = 1e-4 if dtype == torch.float32 else 3e-3
    Cin, Cout, (B, D, H, W) = 32, 4, (2, 5, 13, 9)
    x_ld, x_coff, y_ld, y_coff, vec = HEAD_FWD[layout]
    x = randh(B, D, H, W, Cin, dtype=dtype, seed=14)
    w = (torch.randn(Cout, Cin, 1, 1, 1, generator=torch.Generator().manual_seed(15)) * 0.3).cuda()
    b = torch.randn(Cout, generator=torch.Generator().manual_seed(16)).cuda()
    wp = ops.pack_weight(w, dtype)
    yd = torch.empty(B, D, H, W, Cout, dtype=dtype, device="cuda")
    conv_raw(lib, x, 0, None, 0, wp, yd, 0, None, Cin, Cout, (1, 1, 1), ops.ALGO_DIRECT, bias=b)
    ys = sentinel((B, D, H, W), y_ld, dtype)
    conv_raw(lib, wide(x, x_ld, x_coff), x_coff, None, 0, wp, ys, y_coff, None, Cin, Cout, (1, 1, 1), ops.ALGO_DIRECT, bias=b)
    torch.cuda.synchronize()
    assert_untouched(ys, y_coff, Cout)
    y = ys[..., y_coff:y_coff + Cout]
    same(y, yd, exact=vec, tol=1e-6 if dtype == torch.float32 else 1e-3)
    ref = F.conv3d(nc(x), rnd(w.cpu(), dtype), b.double().cpu())
    assert rel_err(nc(y), ref) < tol


# (x_ld, x_coff, dy_ld, dy_coff, same kernel as the dense call)
HEAD_WGRAD = {"head_dy_vector": (40, 8, 8, 4, True), "head_dy_scalar": (40, 8, 6, 2, False),
              "x_coff4_direct": (36, 4, 8, 4, False)}


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(HEAD_WGRAD))
def test_head_wgrad_sliced(lib, layout, dt):
    ops = lib.ops
    dtype, _ = DTYPES[dt]
    tol = 1e-4 if dtype == torch.float32 else 2e-3
    Cin, Cout, (B, D, H, W) = 32, 4, (2, 5, 12, 9)
    x_ld, x_coff, dy_ld, dy_coff, exact = HEAD_WGRAD[layout]
    x = randh(B, D, H, W, Cin, dtype=dtype, seed=17)
    dy = randh(B, D, H, W, Cout, dtype=dtype, seed=18)
    dwd, dbd = ops.conv3d_wgrad(x, 0, Cin, None, 0, dy, 0, Cout, (1, 1, 1), want_bias=True)
    dws, dbs = ops.conv3d_wgrad(wide(x, x_ld, x_coff), x_coff, Cin, None, 0, wide(dy, dy_ld, dy_coff), dy_coff, Cout,
                                (1, 1, 1), want_bias=True)
    torch.cuda.synchronize()
    same(dws, dwd, exact, tol=1e-5)
    same(dbs, dbd, exact, tol=1e-5)
    wref, bref = _wgrad64(x, None, 0, dy, (1, 1, 1), Cout, bias=True)
    assert rel_err(dws, wref) < tol and rel_err(dbs, bref) < tol


# ----------------------------------------------------------------------------- InstanceNorm family (instnorm.cu)
# (ld - C, coff): VEC=8 needs ld, coff (and C) multiples of 8; the others take the VEC=1 kernels
IN_LAYOUTS = {"vec8": (16, 8), "coff4_vec1": (8, 4), "ld_odd_vec1": (3, 1)}
IN_C, IN_SHAPE = 32, (2, 3, 7, 10)


def _in_case(dt, layout, seed):
    dtype, tol = DTYPES[dt]
    extra, coff = IN_LAYOUTS[layout]
    x = randh(*IN_SHAPE, IN_C, dtype=dtype, scale=2.0, seed=seed) + 0.5
    return dtype, tol, IN_C + extra, coff, layout == "vec8", x


def _in_call(lib, name, *args):
    lib._lib.call(name, *args, lib.ops._stream())


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(IN_LAYOUTS))
def test_instnorm_stats_sliced(lib, layout, dt):
    dtype, _, ld, coff, vec8, x = _in_case(dt, layout, 20)
    B, V, C = IN_SHAPE[0], x[0, ..., 0].numel(), IN_C
    sd, ss = zstats(B, C), zstats(B, C)
    _in_call(lib, "b200seg_instnorm_stats", x.data_ptr(), lib.ops._dt(x), C, 0, B, V, C, sd.data_ptr())
    xs = wide(x, ld, coff)       # every buffer a kernel reads stays referenced until the kernel has run
    _in_call(lib, "b200seg_instnorm_stats", xs.data_ptr(), lib.ops._dt(x), ld, coff, B, V, C, ss.data_ptr())
    torch.cuda.synchronize()
    if vec8:
        assert rel_err(ss, sd) < 1e-12       # same partials, only the order of the fp64 atomics differs
    assert rel_err(ss, stats64(x)) < 1e-5


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(IN_LAYOUTS))
def test_instnorm_apply_sliced(lib, layout, dt, act):
    dtype, tol, ld, coff, vec8, x = _in_case(dt, layout, 21)
    B, V, C = IN_SHAPE[0], x[0, ..., 0].numel(), IN_C
    st = stats64(x)
    yd = torch.empty_like(x)
    _in_call(lib, "b200seg_instnorm_apply", x.data_ptr(), lib.ops._dt(x), C, 0, st.data_ptr(), EPS, act, yd.data_ptr(), C, 0, B, V, C)
    ys = sentinel(IN_SHAPE, ld + 8, dtype)
    xs = wide(x, ld, coff)
    _in_call(lib, "b200seg_instnorm_apply", xs.data_ptr(), lib.ops._dt(x), ld, coff, st.data_ptr(), EPS, act,
             ys.data_ptr(), ld + 8, coff, B, V, C)
    torch.cuda.synchronize()
    assert_untouched(ys, coff, C)
    y = ys[..., coff:coff + C]
    same(y, yd, vec8, tol=1e-6 if dtype == torch.float32 else 1e-3)
    assert rel_err(nc(y), act64(xhat64(x, st), act)) < tol


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(IN_LAYOUTS))
def test_instnorm_bwd_reduce_sliced(lib, layout, dt, act):
    dtype, tol, ld, coff, vec8, x = _in_case(dt, layout, 22)
    B, V, C = IN_SHAPE[0], x[0, ..., 0].numel(), IN_C
    dy = randh(*IN_SHAPE, C, dtype=dtype, seed=23)
    st = stats64(x)
    gd, bd = torch.empty_like(x), zstats(B, C)
    _in_call(lib, "b200seg_instnorm_bwd_reduce", dy.data_ptr(), C, 0, x.data_ptr(), C, 0, lib.ops._dt(x), st.data_ptr(), EPS,
             act, gd.data_ptr(), C, 0, bd.data_ptr(), B, V, C)
    gs, bs = sentinel(IN_SHAPE, ld + 8, dtype), zstats(B, C)
    dys, xs = wide(dy, ld + 16, coff + 8), wide(x, ld, coff)
    _in_call(lib, "b200seg_instnorm_bwd_reduce", dys.data_ptr(), ld + 16, coff + 8, xs.data_ptr(), ld, coff, lib.ops._dt(x), st.data_ptr(), EPS, act, gs.data_ptr(), ld + 8, coff,
             bs.data_ptr(), B, V, C)
    torch.cuda.synchronize()
    assert_untouched(gs, coff, C)
    g = gs[..., coff:coff + C]
    same(g, gd, vec8, tol=1e-6 if dtype == torch.float32 else 1e-3)
    if vec8:
        assert rel_err(bs, bd) < 1e-12
    h = xhat64(x, st)
    gref = rnd(nc(dy) * dact64(h, act), dtype)
    assert rel_err(nc(g), gref) < tol
    bref = torch.stack([gref.sum((2, 3, 4)), (gref * h).sum((2, 3, 4))], -1)
    assert rel_err(bs, bref) < 1e-5


@pytest.mark.parametrize("with_add", [False, True])
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(IN_LAYOUTS))
def test_instnorm_bwd_apply_sliced(lib, layout, dt, with_add):
    dtype, tol, ld, coff, vec8, x = _in_case(dt, layout, 24)
    B, V, C = IN_SHAPE[0], x[0, ..., 0].numel(), IN_C
    g = randh(*IN_SHAPE, C, dtype=dtype, seed=25)
    add = randh(*IN_SHAPE, C, dtype=dtype, seed=26) if with_add else None
    st = stats64(x)
    h = xhat64(x, st)
    bst = torch.stack([nc(g).sum((2, 3, 4)), (nc(g) * h).sum((2, 3, 4))], -1).cuda()
    dt_ = lib.ops._dt(x)
    dd = torch.empty_like(x)
    _in_call(lib, "b200seg_instnorm_bwd_apply", g.data_ptr(), C, 0, x.data_ptr(), C, 0, dt_, st.data_ptr(), bst.data_ptr(), EPS,
             _p(add), C if with_add else 0, 0, dd.data_ptr(), C, 0, B, V, C)
    adds = wide(add, ld + 8, coff) if with_add else None
    ds = sentinel(IN_SHAPE, ld, dtype)
    gw, xs = wide(g, ld + 16, coff), wide(x, ld, coff)
    _in_call(lib, "b200seg_instnorm_bwd_apply", gw.data_ptr(), ld + 16, coff, xs.data_ptr(),
             ld, coff, dt_, st.data_ptr(), bst.data_ptr(), EPS, _p(adds), ld + 8 if with_add else 0, coff,
             ds.data_ptr(), ld, coff, B, V, C)
    torch.cuda.synchronize()
    assert_untouched(ds, coff, C)
    dx = ds[..., coff:coff + C]
    same(dx, dd, vec8, tol=1e-6 if dtype == torch.float32 else 1e-3)
    n = float(V)
    st64 = st.double().cpu()
    r = (1.0 / torch.sqrt(st64[..., 1] / n - (st64[..., 0] / n) ** 2 + EPS))[:, :, None, None, None]
    b64 = bst.double().cpu()
    ref = r * (nc(g) - (b64[..., 0] / n)[:, :, None, None, None] - h * (b64[..., 1] / n)[:, :, None, None, None])
    if with_add:
        ref = ref + nc(add)
    assert rel_err(nc(dx), ref) < tol


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("pair", ["f16_f16", "f32_f16", "f16_f32", "f32_f32"])
@pytest.mark.parametrize("layout", list(IN_LAYOUTS))
def test_copy_channels_sliced(lib, layout, pair, accumulate):
    tx, ty = ({"f16": torch.float16, "f32": torch.float32}[s] for s in pair.split("_"))
    extra, coff = IN_LAYOUTS[layout]
    C = IN_C
    x = randh(*IN_SHAPE, C, dtype=tx, seed=27)
    y0 = randh(*IN_SHAPE, C, dtype=ty, seed=28)
    ys = sentinel(IN_SHAPE, C + extra + 8, ty)
    ys[..., coff:coff + C] = y0
    xs = wide(x, C + extra, coff)
    lib.ops.copy_channels(xs, coff, ys, coff, C, accumulate=accumulate)
    torch.cuda.synchronize()
    assert_untouched(ys, coff, C)
    ref = (x.float() + y0.float() if accumulate else x.float()).to(ty)
    assert torch.equal(ys[..., coff:coff + C], ref)


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("proj", [False, True])
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("layout", list(IN_LAYOUTS))
def test_resblock_out_sliced_r3(lib, layout, dt, proj, act):
    """y = act(IN(r2) + (IN(r3) if stats3 else r3)) and its backward sums, with r3 a slice (r3_ld, r3_coff)."""
    dtype, tol, ld, coff, vec8, r3 = _in_case(dt, layout, 29)
    B, V, C = IN_SHAPE[0], r3[0, ..., 0].numel(), IN_C
    r2 = randh(*IN_SHAPE, C, dtype=dtype, scale=3.0, seed=30)
    dy = randh(*IN_SHAPE, C, dtype=dtype, seed=31)
    st2 = stats64(r2)
    st3 = stats64(r3) if proj else None
    dt_ = lib.ops._dt(r2)
    r3s = wide(r3, ld, coff)
    out = {}
    for name, (t, t_ld, t_coff) in {"dense": (r3, C, 0), "slice": (r3s, ld, coff)}.items():
        y = torch.empty_like(r2)
        _in_call(lib, "b200seg_resblock_out_fwd", r2.data_ptr(), C, st2.data_ptr(), t.data_ptr(), t_ld, t_coff, _p(st3),
                 EPS, act, y.data_ptr(), C, B, V, C, dt_)
        g, sums = torch.empty_like(r2), zstats(B, C, 3)
        _in_call(lib, "b200seg_resblock_out_bwd_reduce", dy.data_ptr(), C, y.data_ptr(), C, r2.data_ptr(), C, st2.data_ptr(),
                 t.data_ptr(), t_ld, t_coff, _p(st3), EPS, act, g.data_ptr(), sums.data_ptr(), B, V, C, dt_)
        out[name] = (y, g, sums)
    torch.cuda.synchronize()
    (yd, gd, sd), (ys, gs, ss) = out["dense"], out["slice"]
    ftol = 1e-6 if dtype == torch.float32 else 1e-3
    same(ys, yd, vec8, ftol)
    same(gs, gd, vec8, ftol)
    if vec8:
        assert rel_err(ss, sd) < 1e-12
    h2 = rnd(xhat64(r2, st2), dtype)
    h3 = rnd(xhat64(r3, st3), dtype) if proj else nc(r3)
    assert rel_err(nc(ys), act64(rnd(h2 + h3, dtype), act)) < tol
    gref = rnd(nc(dy) * dact64(nc(ys), act), dtype)
    assert rel_err(nc(gs), gref) < tol
    x2, x3 = xhat64(r2, st2), (xhat64(r3, st3) if proj else torch.zeros_like(h2))
    sref = torch.stack([gref.sum((2, 3, 4)), (gref * x2).sum((2, 3, 4)), (gref * x3).sum((2, 3, 4))], -1)
    assert rel_err(ss, sref) < 1e-5


# ----------------------------------------------------------------------------- tensor-core routing limits
# both sides of B*Cin = 4096, B*Cout = 2048 and B*Cout = 8192, and the fused ResUNet convolutions that cross 2048 from
# batch 4 / 5 (down4: 256 -> 320 + shortcut = 640; up1: 576 -> 256 + shortcut = 512 and its data gradient 512 -> 576)
ROUTE = [(256, 32, (3, 3, 3), 16), (256, 32, (3, 3, 3), 17), (64, 512, (1, 1, 1), 4), (64, 512, (1, 1, 1), 5),
         (64, 1024, (1, 1, 1), 8), (64, 1024, (1, 1, 1), 9), (16, 2048, (1, 1, 1), 4), (256, 640, (3, 3, 3), 4),
         (576, 512, (3, 3, 3), 5), (512, 576, (3, 3, 3), 5), (768, 3072, (1, 1, 1), 2)]


@pytest.mark.parametrize("Cin,Cout,k,B", ROUTE)
def test_tc_routing_matches_kernel(lib, Cin, Cout, k, B):
    """Every shape routed to the tensor cores runs there with fused statistics, with a residual and in dgrad mode,
    and agrees with the CUDA-core kernel; the others are routed to the CUDA cores."""
    ops = lib.ops
    D, H, W = 2, 5, 3
    tc = B * Cin <= 4096 and B * Cout <= 8192
    assert (ops.conv_algo(Cin, Cout, k, torch.float16, B) == ops.ALGO_TC) == tc
    if not tc:
        return
    taps = k[0] * k[1] * k[2]
    x = randh(B, D, H, W, Cin, seed=32)
    w = (torch.randn(Cout, Cin, *k, generator=torch.Generator().manual_seed(33)) / (Cin * taps) ** 0.5).cuda()
    res = randh(B, D, H, W, Cout, seed=34)
    gx = randh(B, D, H, W, Cout, seed=35)
    xst = stats64(x)
    dg = (gx, 0, stats64(gx), ops.ACT_RELU)
    calls = {"stats": dict(x_stats=xst, act=ops.ACT_RELU), "residual": dict(x_stats=xst, act=ops.ACT_RELU, residual=res),
             "dgrad": dict(x_stats=None, act=ops.ACT_NONE, dgrad_of=dg)}
    wps = {a: ops.pack_weight(w, torch.float16, layout=a) for a in (ops.ALGO_DIRECT, ops.ALGO_TC)}
    for name, kw in calls.items():
        xs, act = kw.pop("x_stats"), kw.pop("act")
        (yd, sd), (yt, st) = (ops.conv3d_fwd(x, 0, Cin, xs, act, wps[a], Cout, k, algo=a, **kw)
                              for a in (ops.ALGO_DIRECT, ops.ALGO_TC))
        torch.cuda.synchronize()
        assert rel_err(yt.float(), yd.float()) < 3e-3, name
        assert rel_err(st, sd) < 1e-3, name


@pytest.mark.parametrize("B", [4, 5])
def test_resunet_amp_batch_crosses_stats_limit(lib, B):
    """ResUNet base 32 (ACDC scales) under AMP at batches where down4's fused conv (B*640) and, from B = 5, up1's
    (B*512) carry more than 2048 output channels per launch, with fused statistics: forward and backward run on the
    tensor cores, gradients are finite and close to the same network in fp32."""
    from oracle.synth import make_volume
    scale = [[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2]]
    kernel = [[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]]
    torch.manual_seed(36)
    net = lib.UNet(1, 32, scale=scale, kernel_size=kernel, num_classes=4, block="BasicBlock", norm="in").cuda()
    img, lab = make_volume(B, 8, 32, 32, 4, seed=37)
    loss_fn = lib.DiceCELoss(weight=torch.tensor([0.5, 1, 1, 1]))
    grads = {}
    for amp in (True, False):
        net.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            loss = loss_fn(net(img.cuda()), lab.cuda())
        (loss * 1024.0).backward()
        grads[amp] = {n: p.grad / 1024.0 for n, p in net.named_parameters()}
    torch.cuda.synchronize()
    assert all(torch.isfinite(g).all() for g in grads[True].values())
    assert global_l2(grads[True], grads[False]) < 0.25
