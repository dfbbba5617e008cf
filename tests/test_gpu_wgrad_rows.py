"""The tensor-core weight gradient stages dy as 32- or 64-channel swizzled voxel rows when min(Cout, 128) is 32, 64 or
128, and x likewise when its Cin tile is 32, 64 or 96; every other width keeps the 16-byte channel planes.  The image
only changes how the operands arrive: the MMAs, their operands and their K order are the same, so dW must not change.

Rows cover each row-image combination (Cin tile 32 / 64 / 96 x min(Cout, 128) 32 / 64 / 128), row images next to plane
images, whole 16x8 tiles and 8-row halves, k 1x1x1 / 1x3x3 / 3x3x3, raw, InstanceNorm + ReLU, InstanceNorm + LeakyReLU
and per-channel (BatchNorm) inputs, channel-sliced x and dy, B = 2, H and W that are not multiples of the tile, and one
CTA per job (S = 1) as well as split-K.

Per row: two calls give the same bits, dW matches a float64 host reference within WG_BAR, and the bytes of dW hash to
what the kernel computed with plane images only (PREVIOUS_CRC, recorded on an H100 80GB HBM3 from the same seeded
inputs).  The inputs and the InstanceNorm sums are made on the host, the sums in float64, so they are the same bits on
every machine.

`python tests/test_gpu_wgrad_rows.py` prints each row's hash."""
import os
import sys
import zlib

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from util import rel_err, wide  # noqa: E402

WG_BAR = 3e-4                                  # tests/test_gpu_tc.py: weight gradient behind the normalising loader
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2
LRELU_SLOPE = 0.01
IN_EPS = 1e-4
K1, K133, K3 = (1, 1, 1), (1, 3, 3), (3, 3, 3)

# name: (Cin, Cout, k, (B, D, H, W), input, x (ld, coff) or None, dy (ld, coff) or None); the comment gives the images
# (x / dy: rows of 32 or 64 channels, or planes) and the staging fill_params picks
ROWS = {
    "x32_dy32_k333_in_relu": (32, 32, K3, (2, 3, 20, 12), "in_relu", None, None),              # r32 / r32, whole
    "x32_dy64_k133_raw_sliced": (32, 64, K133, (1, 4, 20, 12), "raw", (48, 8), (80, 16)),      # r32 / r64
    "x32_dy128_k111_bn": (32, 128, K1, (2, 2, 20, 12), "bn", None, None),                      # r32 / r64 x2
    "x64_dy32_k133_in_lrelu": (64, 32, K133, (2, 3, 20, 12), "in_lrelu", None, None),          # r64 / r32
    "x64_dy64_k333_bn_sliced": (64, 64, K3, (1, 3, 20, 12), "bn", (96, 16), None),             # r64 / r64
    "x64_dy128_k333_in_relu_sliced": (64, 128, K3, (2, 3, 20, 12), "in_relu", None, (160, 32)),  # r64 / r64 x2, whole
    "x128_dy128_k133_raw": (128, 128, K133, (1, 4, 20, 12), "raw", None, None),                # r64 / r64 x2, 2 Cin tiles
    "x96_dy32_k111_in_relu_sliced": (96, 32, K1, (2, 3, 20, 12), "in_relu", (128, 32), None),  # r32 x3 / r32
    "x96_dy64_k133_bn": (96, 64, K133, (1, 3, 20, 12), "bn", None, None),                      # r32 x3 / r64
    "x96_dy128_k333_in_lrelu": (96, 128, K3, (1, 3, 20, 12), "in_lrelu", None, None),          # r32 x3 / r64 x2, halves
    "x192_dy128_k133_raw_sliced": (192, 128, K133, (1, 4, 20, 12), "raw", None, (256, 64)),    # r32 x3 / r64 x2, halves
    "x64_dy256_k333_bn": (64, 256, K3, (2, 2, 20, 12), "bn", None, None),                      # r64 / r64 x2, 2 Cout tiles
    "x64_dy128_k333_in_relu_s1": (64, 128, K3, (1, 1, 12, 8), "in_relu", None, None),          # one voxel tile: S = 1
    "x96_dy64_k111_raw_s1": (96, 64, K1, (1, 1, 16, 8), "raw", None, None),                    # S = 1
    "x64_dy96_k133_in_relu": (64, 96, K133, (2, 3, 20, 12), "in_relu", None, None),            # r64 / planes
    "x48_dy64_k333_raw": (48, 64, K3, (1, 3, 20, 12), "raw", None, None),                      # planes / r64
    "x16_dy32_k111_in_lrelu_sliced": (16, 32, K1, (2, 3, 20, 12), "in_lrelu", (32, 8), (48, 8)),  # planes / r32
}

PREVIOUS_CRC = {
    "x32_dy32_k333_in_relu": 0x9925ba71,
    "x32_dy64_k133_raw_sliced": 0x3dbe3c1e,
    "x32_dy128_k111_bn": 0xbe621857,
    "x64_dy32_k133_in_lrelu": 0x364743db,
    "x64_dy64_k333_bn_sliced": 0xf8304204,
    "x64_dy128_k333_in_relu_sliced": 0x73d773c7,
    "x128_dy128_k133_raw": 0xcdccef34,
    "x96_dy32_k111_in_relu_sliced": 0xdc4f59b1,
    "x96_dy64_k133_bn": 0x77465afd,
    "x96_dy128_k333_in_lrelu": 0x16de61e0,
    "x192_dy128_k133_raw_sliced": 0xb57122f5,
    "x64_dy256_k333_bn": 0x91d8bdd6,
    "x64_dy128_k333_in_relu_s1": 0x3108e072,
    "x96_dy64_k111_raw_s1": 0x576529e2,
    "x64_dy96_k133_in_relu": 0xbb777a84,
    "x48_dy64_k333_raw": 0x490d939a,
    "x16_dy32_k111_in_lrelu_sliced": 0x9bb598d2,
}


def _inputs(name):
    Cin, Cout, k, (B, D, H, W), kind, xs, dys = ROWS[name]
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) & 0x7fffffff)
    x = torch.randn(B, D, H, W, Cin, generator=g).half()
    dy = torch.randn(B, D, H, W, Cout, generator=g).half()
    stats = affine = None
    if kind.startswith("in_"):
        d = x.double().flatten(1, 3)
        stats = torch.stack([d.sum(1), (d * d).sum(1)], -1).contiguous()
    elif kind == "bn":
        affine = torch.stack([0.5 + torch.rand(Cin, generator=g), torch.rand(Cin, generator=g) - 0.5], -1).contiguous()
    act = {"raw": ACT_NONE, "in_relu": ACT_RELU, "in_lrelu": ACT_LRELU, "bn": ACT_RELU}[kind]
    return x, dy, stats, affine, act


def _wgrad(name):
    from b200seg import _lib, ops
    Cin, Cout, k, (B, D, H, W), kind, xs, dys = ROWS[name]
    x, dy, stats, affine, act = _inputs(name)
    x_ld, x_coff = xs or (Cin, 0)
    dy_ld, dy_coff = dys or (Cout, 0)
    xb, dyb = wide(x, x_ld, x_coff).cuda(), wide(dy, dy_ld, dy_coff).cuda()
    if affine is None:
        dw, _ = ops.conv3d_wgrad(xb, x_coff, Cin, None if stats is None else stats.cuda(), act, dyb, dy_coff, Cout, k,
                                 algo=_lib.ALGO_TC)
    else:
        aff = affine.cuda()
        dw = torch.zeros(Cout, Cin, *k, dtype=torch.float32, device="cuda")
        lib = _lib.load()
        ws_bytes = lib.b200seg_conv3d_wgrad_pc_workspace(x_ld, x_coff, 1, dy_ld, dy_coff, 0, B, D, H, W, Cin, Cout, *k,
                                                         ops._dt(xb), _lib.ALGO_TC)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda") if ws_bytes else None
        _lib.call("b200seg_conv3d_wgrad_pc", xb.data_ptr(), x_ld, x_coff, aff.data_ptr(), act, dyb.data_ptr(), dy_ld,
                  dy_coff, dw.data_ptr(), None, B, D, H, W, Cin, Cout, *k, ops._dt(xb), _lib.ALGO_TC,
                  ops._p(ws), ws_bytes, ops._stream())
    torch.cuda.synchronize()
    return dw


def _reference(name):
    """dW in float64 on the host, from the fp16 operand a = act(x * s + t) the kernel's loader makes"""
    Cin, Cout, k, _, kind, _, _ = ROWS[name]
    x, dy, stats, affine, act = _inputs(name)
    xf = x.float()
    if stats is not None:
        n = x.shape[1] * x.shape[2] * x.shape[3]
        m = stats[..., 0] / n
        var = (stats[..., 1] / n - m * m).clamp_min(0.0)
        mean, rstd = m.float(), (1.0 / torch.sqrt(var + IN_EPS)).float()
        xf = xf * rstd[:, None, None, None, :] + (-mean * rstd)[:, None, None, None, :]
    elif affine is not None:
        xf = xf * affine[:, 0] + affine[:, 1]
    if act == ACT_RELU:
        xf = xf.clamp_min(0.0)
    elif act == ACT_LRELU:
        xf = torch.where(xf > 0, xf, LRELU_SLOPE * xf)
    a = xf.half().double().permute(0, 4, 1, 2, 3)
    g = dy.double().permute(0, 4, 1, 2, 3)
    return torch.nn.grad.conv3d_weight(a, (Cout, Cin, *k), g, padding=tuple(v // 2 for v in k))


def _crc(dw):
    return zlib.crc32(dw.cpu().contiguous().numpy().tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(ROWS))
def test_wgrad_rows_keep_the_bits(row, record_property):
    first, second = _wgrad(row), _wgrad(row)
    assert torch.equal(first, second)
    err = rel_err(first, _reference(row))
    record_property("wg_err", err)
    assert err < WG_BAR, err
    assert _crc(first) == PREVIOUS_CRC[row], "dW differs from the plane-image kernel's result: %08x" % _crc(first)


if __name__ == "__main__":
    print("{" + ", ".join('"%s": 0x%08x' % (r, _crc(_wgrad(r))) for r in ROWS) + "}")
