"""The side operand of the tensor-core convolution epilogue (csrc/conv_tc.cu): the residual of a forward and the
pre-norm input `gx` behind the activation mask of a data gradient arrive as one tensor-TMA box per output tile in a
ring of shared-memory slots (two slots for NT <= 64, one above), filled by their own producer warp up to a tile or two
ahead of the epilogue.

Each row runs a forward with IN + ReLU loader and residual, and a data gradient with the ReLU mask of `gx`, against
float64 with the bars of test_gpu_tc.py, and checks that a second identical call stores the same bits.  The rows cover
every N tile on both slot counts (NT 16 / 32 / 48 / 64 with two slots, 80 and 128 with one, and later N tiles of one
launch for 80 and 128), ragged 16 x 8 tiles and B = 2, a grid in which some CTAs own three tiles and others two (the
ring wraps at a different tile on each), and residual / `gx` read as channel slices at a non-zero offset of a wider
tensor.
"""
import pytest
import torch

from test_gpu_tc import ACT_RELU, FWD_BAR, MASK_MARGIN, STATS_BAR, _masked_err, conv64, dact64, loader64, nc, randf, randh, seed_of, \
    stats64, xhat64
from util import rel_err

gpu = pytest.mark.gpu
K133, K333 = (1, 3, 3), (3, 3, 3)
RAGGED = (2, 3, 20, 12)          # B = 2, H and W not multiples of the 16 x 8 tile

ROWS = {  # name: Cin, Cout, k, (B, D, H, W), channel offset of the side operand inside a wider tensor
    "nt16": (16, 16, K333, RAGGED, 0),
    "nt32": (32, 32, K133, RAGGED, 0),
    "nt48": (48, 48, K333, RAGGED, 0),
    "nt64": (64, 64, K133, RAGGED, 0),
    "nt80_two_ntiles": (32, 160, K333, RAGGED, 0),
    "nt128_two_ntiles": (64, 256, K133, RAGGED, 0),
    "nt32_odd_tiles_per_cta": (32, 32, K133, (1, 10, 48, 88), 0),     # 330 tiles on 132 CTAs: 3 or 2 each
    "nt32_slice": (32, 32, K133, RAGGED, 8),
    "nt64_slice": (64, 64, K333, RAGGED, 16),
    "nt128_slice": (128, 128, K133, RAGGED, 24),
}


def _side(shape, C, coff, seed):
    """a [B, D, H, W, C] operand, stored as channels coff .. coff + C of a wider tensor when coff > 0"""
    B, D, H, W = shape
    full = randh(B, D, H, W, C + 2 * coff if coff else C, seed=seed)
    return full, full[..., coff:coff + C]


def _launch(mode, x, xst, w, Cin, Cout, k, side_full, coff):
    from b200seg import ops, _lib
    wp = ops.pack_weight(w, torch.float16, layout=_lib.ALGO_TC)
    if mode == "res":
        return ops.conv3d_fwd(x, 0, Cin, xst, ACT_RELU, wp, Cout, k, residual=side_full, r_coff=coff, algo=_lib.ALGO_TC)
    gst = stats64(side_full[..., coff:coff + Cout])
    return ops.conv3d_fwd(x, 0, Cin, None, 0, wp, Cout, k, dgrad_of=(side_full, coff, gst, ACT_RELU), algo=_lib.ALGO_TC)


@gpu
@pytest.mark.parametrize("mode", ["res", "dgrad"])
@pytest.mark.parametrize("row", list(ROWS))
def test_side_tile_epilogue(row, mode, record_property):
    from b200seg import ops, _lib
    Cin, Cout, k, shape, coff = ROWS[row]
    B = shape[0]
    assert ops.conv_algo(Cin, Cout, k, torch.float16, B) == _lib.ALGO_TC
    seed = seed_of(row + mode)
    taps = k[0] * k[1] * k[2]
    x = randh(B, *shape[1:], Cin, seed=seed)
    w = randf(Cout, Cin, *k, seed=seed + 1) / (Cin * taps) ** 0.5
    side_full, side = _side(shape, Cout, coff, seed + 2)
    xst = stats64(x) if mode == "res" else None
    y1, st1 = _launch(mode, x, xst, w, Cin, Cout, k, side_full, coff)
    y2, st2 = _launch(mode, x, xst, w, Cin, Cout, k, side_full, coff)
    torch.cuda.synchronize()
    assert torch.equal(y1.view(torch.int16), y2.view(torch.int16)), "two identical calls stored different bits"

    if mode == "res":
        ref = conv64(loader64(x, xst, ACT_RELU), w.half(), k).half().double() + nc(side)
        keep, h = torch.ones_like(ref, dtype=torch.bool), None
    else:
        h = xhat64(side, stats64(side))
        ref = conv64(nc(x), w.half(), k) * dact64(h, ACT_RELU)
        keep = h.abs() >= MASK_MARGIN
    y = nc(y1)
    err = _masked_err(y, ref, keep)
    record_property("fwd_err", err)
    assert err < FWD_BAR, err
    sref = stats64(y1) if h is None else torch.stack([y.sum((2, 3, 4)), (y * h).sum((2, 3, 4))], -1)
    serr = max(rel_err(st1, sref), rel_err(st2, sref))
    record_property("stats_err", serr)
    assert serr < STATS_BAR, serr

