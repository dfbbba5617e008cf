"""GPU: max-pool and trilinear upsample (align_corners) kernels of pool_upsample.cu against PyTorch in fp64.

Every call goes through the C ABI with explicit (ld, coff) channel slices, as the models use them: a sliced input is a
wider buffer whose other channels hold +-POISON, a sliced output a wider buffer whose other channels must keep the
sentinel bit for bit.  Both kernels move 8 channels per thread (VEC = 8) when C, ld and coff are multiples of 8, and
one otherwise (VEC = 1, at most 256 channels).  The oracle is F.max_pool3d / F.interpolate(mode="trilinear",
align_corners=True) in fp64 on the device, with autograd, on the same fp16-rounded inputs.  For fp16 and fp32 tensors
ATen computes the source coordinate src = scale * o, scale = (in - 1) / (out - 1), in fp32, and so does the kernel;
at 979 -> 1958 that alone moves an fp32 result by 5e-5 of its range.  The upsample is therefore checked against the
same interpolation restated in fp64 with those fp32 coordinates (interp64), which is itself checked against the fp64
F.interpolate to the coordinates' rounding.  Bars:
  * max-pool: values and gradient bit-equal (ties go to the first maximum in (d, h, w) order, as in torch);
  * upsample forward: fp32 rel_err 1e-5; fp16 within one fp16 ulp of the fp64 value, plus the fp32 evaluation's own
    error (a few fp32 ulps of the inputs, visible only where the result is near 0);
  * upsample backward: fp32 rel_err 1e-5, fp16 3e-3;
  * InstanceNorm sums of the stored output: rel_err 1e-5 against the fp64 sums.
The backward gathers per axis through tables of at most 12 output taps (upsampling factors up to ~4.5), held in
shared memory at sizeof(AxisTab) = 100 bytes per input index, with an opt-in above 48 KB and a limit of 96 KB.
"""
import re

import pytest
import torch
import torch.nn.functional as F

from util import SENTINEL, assert_untouched, launched_kernels, sentinel, wide

pytestmark = pytest.mark.gpu

TAB_BYTES = 100        # sizeof(AxisTab): n + 12 output indices + 12 weights


@pytest.fixture(scope="module")
def lib():
    import b200seg
    from b200seg import _lib, ops  # noqa: F401
    assert _lib.load().b200seg_check_device() == 0, "not an H100"
    return b200seg


def rand(lead, C, dtype, seed, quantize=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(*lead, C, generator=g, device="cuda")
    if quantize:                   # quarter steps: many exact ties inside a pooling window
        x = (x * 4).round() / 4
    return x.to(dtype)


def rel_err(a, b):
    """util.rel_err on the device: the benchmark rows compare up to 2.6e8 elements"""
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def nc64(t):
    """[B, D, H, W, C] -> [B, C, D, H, W] fp64"""
    return t.double().permute(0, 4, 1, 2, 3)


def cl(t):
    return t.permute(0, 2, 3, 4, 1)


def stats64(t):
    d = t.double().flatten(1, 3)
    return torch.stack([d.sum(1), (d * d).sum(1)], -1)


def zstats(B, C):
    return torch.zeros(B, C, 2, dtype=torch.float64, device="cuda")


def fp16_ulp(r):
    _, e = torch.frexp(r)
    return torch.ldexp(torch.ones_like(r), (e - 11).clamp_min(-24))


def assert_fwd_close(y, ref, x):
    if y.dtype == torch.float32:
        assert rel_err(y, ref) < 1e-5
    else:
        err = (y.double() - ref).abs()
        bar = fp16_ulp(ref) + 2.0 ** -20 * x.double().abs().max()
        assert (err <= bar).all(), (err - bar).max().item()


def axis_weights(n_in, n_out):
    """[n_out, n_in] fp64 matrix of 1-D linear interpolation with align_corners=True, from fp32 source coordinates"""
    f32 = lambda v: torch.tensor(float(v), dtype=torch.float32)      # noqa: E731
    scale = f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0)
    s = scale * torch.arange(n_out, dtype=torch.float32)
    i0 = s.long().clamp_max(n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = s - i0.float()
    l0 = 1 - l1
    A = torch.zeros(n_out, n_in, dtype=torch.float64)
    o = torch.arange(n_out)
    A.index_put_((o, i0), l0.double(), accumulate=True)
    A.index_put_((o, i1), l1.double(), accumulate=True)
    return A.cuda()


def interp64(x, dst):
    """trilinear (align_corners=True) upsample of x [B, D, H, W, C] (fp64) to dst, one axis at a time"""
    _, Di, Hi, Wi, _ = x.shape
    y = torch.einsum("bdhwc,vw->bdhvc", x, axis_weights(Wi, dst[2]))
    y = torch.einsum("bdhwc,vh->bdvwc", y, axis_weights(Hi, dst[1]))
    return torch.einsum("bdhwc,vd->bvhwc", y, axis_weights(Di, dst[0]))


# ----------------------------------------------------------------------------- launchers (C ABI)
def maxpool_fwd(lib, x, x_coff, C, y, y_coff, idx, st, shape, scale):
    from b200seg import ops
    B, D, H, W = shape
    lib._lib.call("b200seg_maxpool3d_fwd", x.data_ptr(), x.shape[-1], x_coff, y.data_ptr(), y.shape[-1], y_coff,
                  idx.data_ptr(), None if st is None else st.data_ptr(), B, D, H, W, C, *scale, ops._dt(x), ops._stream())


def maxpool_bwd(lib, dy, dy_coff, C, idx, dx, dx_coff, shape, scale):
    from b200seg import ops
    B, D, H, W = shape
    lib._lib.call("b200seg_maxpool3d_bwd", dy.data_ptr(), dy.shape[-1], dy_coff, idx.data_ptr(), dx.data_ptr(),
                  dx.shape[-1], dx_coff, B, D, H, W, C, *scale, ops._dt(dy), ops._stream())


def upsample_fwd(lib, x, x_coff, C, y, y_coff, st, src, dst):
    from b200seg import ops
    lib._lib.call("b200seg_upsample_trilinear_fwd", x.data_ptr(), x.shape[-1], x_coff, y.data_ptr(), y.shape[-1], y_coff,
                  None if st is None else st.data_ptr(), x.shape[0], *src, *dst, C, ops._dt(x), ops._stream())


def upsample_bwd(lib, dy, dy_coff, C, dx, dx_coff, src, dst, accumulate=0):
    from b200seg import ops
    lib._lib.call("b200seg_upsample_trilinear_bwd", dy.data_ptr(), dy.shape[-1], dy_coff, dx.data_ptr(), dx.shape[-1],
                  dx_coff, accumulate, dx.shape[0], *src, *dst, C, ops._dt(dy), ops._stream())


# ----------------------------------------------------------------------------- checks
def check_maxpool(lib, B, C, spatial, scale, dtype, x_lay, y_lay, seed=0):
    """x_lay / y_lay = (ld, coff) of the input / output buffers; the backward uses y_lay for dy and x_lay for dx"""
    (x_ld, x_coff), (y_ld, y_coff) = x_lay, y_lay
    D, H, W = spatial
    sd, sh, sw = scale
    Do, Ho, Wo = D // sd, H // sh, W // sw
    xd = rand((B, D, H, W), C, dtype, seed, quantize=True)
    x = wide(xd, x_ld, x_coff)
    y = sentinel((B, Do, Ho, Wo), y_ld, dtype)
    idx = torch.empty(B, Do, Ho, Wo, C, dtype=torch.uint8, device="cuda")
    st = zstats(B, C)
    maxpool_fwd(lib, x, x_coff, C, y, y_coff, idx, st, (B, D, H, W), scale)
    x64 = nc64(xd).requires_grad_(True)
    yo = F.max_pool3d(x64, scale)
    yk = y[..., y_coff:y_coff + C]
    assert torch.equal(yk, cl(yo.detach()).to(dtype))
    assert_untouched(y, y_coff, C)
    assert rel_err(st, stats64(yk)) < 1e-5

    dyd = rand((B, Do, Ho, Wo), C, dtype, seed + 1)
    dy = wide(dyd, y_ld, y_coff)
    dx = sentinel((B, D, H, W), x_ld, dtype)
    maxpool_bwd(lib, dy, y_coff, C, idx, dx, x_coff, (B, D, H, W), scale)
    yo.backward(nc64(dyd))
    g = cl(x64.grad).to(dtype)
    covered = (slice(None), slice(0, Do * sd), slice(0, Ho * sh), slice(0, Wo * sw))
    assert torch.equal(dx[covered][..., x_coff:x_coff + C], g[covered])
    # the windows' remainder is not written: MaxPoolFn zero-fills dx when the shape does not divide
    outside = torch.ones(B, D, H, W, dtype=torch.bool, device="cuda")
    outside[covered] = False
    assert (dx[outside] == SENTINEL).all()
    assert_untouched(dx, x_coff, C)


def check_upsample(lib, B, C, src, dst, dtype, x_lay, y_lay, seed=0, accumulate=False):
    """x_lay = (ld, coff) of the low-resolution input (and of dx), y_lay of the output (and of dy)"""
    (x_ld, x_coff), (y_ld, y_coff) = x_lay, y_lay
    xd = rand((B, *src), C, dtype, seed)
    x = wide(xd, x_ld, x_coff)
    y = sentinel((B, *dst), y_ld, dtype)
    st = zstats(B, C)
    upsample_fwd(lib, x, x_coff, C, y, y_coff, st, src, dst)
    x64 = xd.double().requires_grad_(True)
    yo = interp64(x64, dst)
    yt = F.interpolate(nc64(xd), size=tuple(dst), mode="trilinear", align_corners=True)
    assert rel_err(yo.detach(), cl(yt)) < 6 * 2.0 ** -23 * max(max(src) - 1, 1) * 2      # |x| < 6 sigma
    del yt
    yk = y[..., y_coff:y_coff + C]
    assert_fwd_close(yk, yo.detach(), xd)
    assert_untouched(y, y_coff, C)
    assert rel_err(st, stats64(yk)) < 1e-5

    dyd = rand((B, *dst), C, dtype, seed + 1)
    dy = wide(dyd, y_ld, y_coff)
    dx = sentinel((B, *src), x_ld, dtype)
    if accumulate:
        dx0 = rand((B, *src), C, dtype, seed + 2)
        dx[..., x_coff:x_coff + C] = dx0
    upsample_bwd(lib, dy, y_coff, C, dx, x_coff, src, dst, int(accumulate))
    yo.backward(dyd.double())
    g = x64.grad
    if accumulate:
        g = g + dx0.double()
    assert rel_err(dx[..., x_coff:x_coff + C], g) < (1e-5 if dtype == torch.float32 else 3e-3)
    assert_untouched(dx, x_coff, C)


# ----------------------------------------------------------------------------- dispatch
LAYOUTS = {                 # (ld, coff) as a function of C; VEC = 8 needs C, ld and coff all multiples of 8
    "dense": lambda C: (C, 0),
    "slice8": lambda C: (C + 16, 8),
    "coff3": lambda C: (C + 8, 3),
    "ld_odd": lambda C: (C + 3, 0),
}
DTYPES = [torch.float32, torch.float16]


def _vec8(C, layout):
    ld, coff = LAYOUTS[layout](C)
    return C % 8 == 0 and ld % 8 == 0 and coff % 8 == 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("C", [3, 14, 16, 40, 256, 320])
def test_maxpool_dispatch(lib, C, layout, dtype):
    """2x2x2 pooling of a 5x7x6 volume (no axis divides): VEC 8 for C = 16, 40, 256, 320 on 8-aligned slices,
    VEC 1 for the rest; VEC 1 above 256 channels is refused"""
    lay = LAYOUTS[layout](C)
    if not _vec8(C, layout) and C > 256:
        with pytest.raises(lib.B200SegError):
            check_maxpool(lib, 2, C, (5, 7, 6), (2, 2, 2), dtype, lay, lay)
        return
    check_maxpool(lib, 2, C, (5, 7, 6), (2, 2, 2), dtype, lay, lay, seed=C)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("C", [3, 14, 16, 40, 256, 320])
def test_upsample_dispatch(lib, C, layout, dtype):
    lay = LAYOUTS[layout](C)
    if not _vec8(C, layout) and C > 256:
        with pytest.raises(lib.B200SegError):
            check_upsample(lib, 2, C, (3, 4, 5), (6, 7, 9), dtype, lay, lay)
        return
    check_upsample(lib, 2, C, (3, 4, 5), (6, 7, 9), dtype, lay, lay, seed=C)


def test_vec1_above_256_channels_raises(lib):
    C, (ld, coff), dt = 257, (257, 0), torch.float16
    x = torch.zeros(1, 4, 4, 4, ld, dtype=dt, device="cuda")
    y = torch.zeros(1, 2, 2, 2, ld, dtype=dt, device="cuda")
    idx = torch.zeros(1, 2, 2, 2, C, dtype=torch.uint8, device="cuda")
    up = torch.zeros(1, 8, 8, 8, ld, dtype=dt, device="cuda")
    for fn in (lambda: maxpool_fwd(lib, x, coff, C, y, coff, idx, None, (1, 4, 4, 4), (2, 2, 2)),
               lambda: maxpool_bwd(lib, y, coff, C, idx, x, coff, (1, 4, 4, 4), (2, 2, 2)),
               lambda: upsample_fwd(lib, x, coff, C, up, coff, None, (4, 4, 4), (8, 8, 8)),
               lambda: upsample_bwd(lib, up, coff, C, x, coff, (4, 4, 4), (8, 8, 8))):
        with pytest.raises(lib.B200SegError):
            fn()
    torch.cuda.synchronize()


_KERNEL = re.compile(r"(maxpool_fwd|maxpool_bwd|upsample_fwd|upsample_bwd)_kernel"
                     r"(?:<\s*(?:__half|float)\s*,\s*(?:\(int\))?\s*(\d+)\s*>|I(?:6__half|f)Li(\d+)EE)")


def run_vec_path_rows():
    import b200seg
    for layout in ("slice8", "coff3", "ld_odd"):
        lay = LAYOUTS[layout](16)
        check_maxpool(b200seg, 1, 16, (2, 4, 4), (1, 2, 2), torch.float16, lay, lay)
        check_upsample(b200seg, 1, 16, (2, 2, 3), (3, 4, 5), torch.float16, lay, lay)


def test_pool_upsample_vec_paths_launch():
    """the dispatch rows above reach both VEC = 8 and VEC = 1 in each of the four kernels"""
    seen = set()
    for name in launched_kernels("test_gpu_pool_upsample", "run_vec_path_rows"):
        m = _KERNEL.search(name)
        if m:
            seen.add((m.group(1), int(m.group(2) or m.group(3))))
    expected = {(k, v) for k in ("maxpool_fwd", "maxpool_bwd", "upsample_fwd", "upsample_bwd") for v in (1, 8)}
    assert seen == expected, sorted(expected ^ seen)


# ----------------------------------------------------------------------------- benchmark rows
def _levels(top, scales):
    dims = [tuple(top)]
    for s in scales:
        dims.append(tuple(d // f for d, f in zip(dims[-1], s)))
    return dims


RESUNET = {       # workload: (B, top volume, per-level pooling scales), bench.py WORKLOADS, channels 32/64/128/256/320
    "resunet_acdc_128": (1, (128, 128, 128), [(1, 2, 2), (1, 2, 2), (2, 2, 2), (2, 2, 2)]),
    "resunet_iso_128": (1, (128, 128, 128), [(2, 2, 2)] * 4),
    "resunet_kits_160": (2, (160, 160, 80), [(2, 2, 2)] * 4),
}
CH = [32, 64, 128, 256, 320]        # also medformer_bcv_96's: base 32, chan_num[0:4] = 64, 128, 256, 320
MEDFORMER_SCALES = [(1, 2, 2), (1, 2, 2), (2, 2, 2), (2, 2, 2)]


@pytest.mark.parametrize("level", range(4))
@pytest.mark.parametrize("workload", list(RESUNET))
def test_maxpool_benchmark_rows(lib, workload, level):
    B, top, scales = RESUNET[workload]
    dims = _levels(top, scales)
    C = CH[level]
    check_maxpool(lib, B, C, dims[level], scales[level], torch.float16, (C, 0), (C, 0), seed=level)


@pytest.mark.parametrize("up", [1, 2, 3, 4])
@pytest.mark.parametrize("workload", list(RESUNET))
def test_upcat_benchmark_rows(lib, workload, up):
    """up_block k upsamples level 5-k (CH[5-k] channels: the bottom level, then each up_block's output) into the concat
    buffer after the skip channels of level 4-k (cat([skip, up]): up1 writes 320 channels at offset 256 of 576)"""
    B, top, scales = RESUNET[workload]
    dims = _levels(top, scales)
    lo, hi = 5 - up, 4 - up
    Cl, Cs = CH[lo], CH[hi]
    check_upsample(lib, B, Cl, dims[lo], dims[hi], torch.float16, (Cl, 0), (Cs + Cl, Cs), seed=up)


@pytest.mark.parametrize("up", [1, 2, 3, 4])
def test_upcat_medformer_rows(lib, up):
    """medformer_bcv_96 up_block k: cat([up, skip]), the upsampled channels first (coff 0)"""
    dims = _levels((96, 96, 96), MEDFORMER_SCALES)
    lo, hi = 5 - up, 4 - up
    Cl, Cs = CH[lo], CH[hi]
    check_upsample(lib, 1, Cl, dims[lo], dims[hi], torch.float16, (Cl, 0), (Cs + Cl, 0), seed=up)


def test_upsample_medformer_aux(lib):
    """MedFormer's auxiliary head: 16 padded class channels from 96x24x24 to the 96^3 crop (23/95 in H and W, close to
    the tap limit)"""
    check_upsample(lib, 1, 16, (96, 24, 24), (96, 96, 96), torch.float16, (16, 0), (16, 0), seed=9)


# ----------------------------------------------------------------------------- geometry
GEOMETRY = {
    "x2": ((3, 4, 5), (6, 8, 10)),
    "x1_2_2": ((4, 3, 5), (4, 6, 10)),
    "non_integer": ((3, 5, 7), (7, 12, 13)),
    "identity": ((4, 5, 6), (4, 5, 6)),
    "downsample": ((12, 4, 3), (5, 7, 3)),
    "near_integer": ((24, 3, 2), (96, 5, 3)),      # scale * o lands next to an integer for many o
    "to_one": ((5, 3, 4), (1, 6, 4)),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [16, 5])
@pytest.mark.parametrize("geom", list(GEOMETRY))
def test_upsample_geometry(lib, geom, C, dtype):
    src, dst = GEOMETRY[geom]
    check_upsample(lib, 2, C, src, dst, dtype, (C, 0), (C, 0), seed=len(geom))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [16, 5])
@pytest.mark.parametrize("n", [2, 12, 13, 16])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_upsample_length_one_axis(lib, axis, n, C, dtype):
    """an input axis of length 1 broadcast to n outputs: its gradient is the sum over all n, whatever n is"""
    src, dst = [3, 4, 5], [5, 7, 9]
    src[axis], dst[axis] = 1, n
    check_upsample(lib, 2, C, tuple(src), tuple(dst), dtype, (C, 0), (C, 0), seed=n)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", ["slice8", "coff3"])
def test_upsample_bwd_accumulate(lib, layout, dtype):
    """accumulate = 1 adds the gradient onto what dx holds"""
    lay = LAYOUTS[layout](16)
    check_upsample(lib, 2, 16, (3, 5, 7), (7, 12, 13), dtype, lay, lay, seed=3, accumulate=True)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [8, 16, 5])
@pytest.mark.parametrize("shape", [(4, 6, 9), (3, 9, 4), (6, 5, 5)])
def test_maxpool_geometry(lib, shape, C, dtype):
    """pooling scales (2, 2, 2), (1, 2, 2) and (2, 3, 1) on shapes that divide in some axes and not in others"""
    for scale in [(2, 2, 2), (1, 2, 2), (2, 3, 1)]:
        check_maxpool(lib, 2, C, shape, scale, dtype, (C, 0), (C, 0), seed=C)


# ----------------------------------------------------------------------------- limits
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_upsample_bwd_above_tap_limit_raises(lib, axis):
    """12 -> 96 needs 18 taps per input index along that axis: refused, never a partial sum"""
    src, dst = [3, 4, 5], [5, 7, 9]
    src[axis], dst[axis] = 12, 96
    dy = torch.zeros(1, *dst, 8, dtype=torch.float16, device="cuda")
    dx = torch.zeros(1, *src, 8, dtype=torch.float16, device="cuda")
    with pytest.raises(lib.B200SegError):
        upsample_bwd(lib, dy, 0, 8, dx, 0, tuple(src), tuple(dst))
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Wi", [500, 979])
def test_upsample_bwd_large_tables(lib, Wi, dtype):
    """Di + Hi + Wi = 504 and 983: the tables take more than the default 48 KB of shared memory (opt-in path), the
    second one the most that fits under the 96 KB limit"""
    src, dst = (2, 2, Wi), (3, 3, 2 * Wi)
    assert 48 * 1024 < TAB_BYTES * sum(src) <= 96 * 1024
    check_upsample(lib, 1, 8, src, dst, dtype, (8, 0), (8, 0), seed=Wi)


def test_upsample_bwd_tables_above_limit_raise(lib):
    src, dst = (2, 2, 980), (3, 3, 1960)
    assert TAB_BYTES * sum(src) > 96 * 1024
    dy = torch.zeros(1, *dst, 8, dtype=torch.float16, device="cuda")
    dx = torch.zeros(1, *src, 8, dtype=torch.float16, device="cuda")
    with pytest.raises(lib.B200SegError):
        upsample_bwd(lib, dy, 0, 8, dx, 0, src, dst)
    torch.cuda.synchronize()
