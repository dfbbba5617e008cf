"""The tensor-core weight gradient stages its operands with tensor TMA into a ring sized from the shape: whole 16x8
voxel tiles, or two 8-row halves per tile where fewer than 4 whole tiles fit in shared memory.  Either way every
accumulator sees the same MMAs in the same K order, so dW must not depend on how the tiles arrive.

Per row: two calls give the same bits, dW matches the CUDA-core kernel (ALGO_DIRECT) within WG_BAR, and the bytes of dW
hash to what the kernel computed before the TMA loader replaced per-thread cp.async staging (PREVIOUS_CRC, recorded on
an H100 80GB HBM3 from the same seeded inputs).  The InstanceNorm sums are computed on the host in float64, so the
inputs are the same bits on every machine.

`python tests/test_gpu_wgrad_staging.py` prints each row's hash."""
import os
import sys
import zlib

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from util import rel_err  # noqa: E402

WG_BAR = 3e-4                                  # tests/test_gpu_tc.py: weight gradient behind the normalising loader
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2
K3 = (3, 3, 3)

ROWS = {   # name: (Cin, Cout, k, (B, D, H, W), act, InstanceNorm statistics); the comment gives the staging fill_params picks
    "whole_relu": (64, 128, K3, (2, 3, 20, 12), ACT_RELU, True),              # 16x8 tiles, 4 stages
    "half_relu": (96, 128, K3, (1, 3, 20, 12), ACT_RELU, True),               # 8-row halves, 6 stages
    "half_raw": (112, 128, (1, 3, 3), (1, 4, 32, 16), ACT_NONE, False),       # halves consumed straight off the TMA
    "tail_lrelu": (16, 16, (1, 1, 1), (2, 3, 20, 12), ACT_LRELU, True),       # A descriptor reads past the ring
}

PREVIOUS_CRC = {"whole_relu": 0xb71149f9, "half_relu": 0xd9bf182e, "half_raw": 0x9a7813c5, "tail_lrelu": 0x60145183}


def _inputs(name):
    Cin, Cout, k, (B, D, H, W), act, stats = ROWS[name]
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) & 0x7fffffff)
    x = torch.randn(B, D, H, W, Cin, generator=g).half()
    dy = torch.randn(B, D, H, W, Cout, generator=g).half()
    st = None
    if stats:
        d = x.double().flatten(1, 3)
        st = torch.stack([d.sum(1), (d * d).sum(1)], -1).contiguous().cuda()
    return x.cuda(), st, act, dy.cuda(), Cin, Cout, k


def _wgrad(name, algo):
    from b200seg import ops
    x, st, act, dy, Cin, Cout, k = _inputs(name)
    dw, _ = ops.conv3d_wgrad(x, 0, Cin, st, act, dy, 0, Cout, k, algo=algo)
    torch.cuda.synchronize()
    return dw


def _crc(dw):
    return zlib.crc32(dw.cpu().contiguous().numpy().tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(ROWS))
def test_wgrad_staging_keeps_the_bits(row, record_property):
    from b200seg import _lib
    first, second = _wgrad(row, _lib.ALGO_TC), _wgrad(row, _lib.ALGO_TC)
    assert torch.equal(first, second)
    err = rel_err(first, _wgrad(row, _lib.ALGO_DIRECT))
    record_property("wg_err", err)
    assert err < WG_BAR, err
    assert _crc(first) == PREVIOUS_CRC[row], "dW differs from the kernel's previous result: %08x" % _crc(first)


if __name__ == "__main__":
    from b200seg import _lib
    print({r: "0x%08x" % _crc(_wgrad(r, _lib.ALGO_TC)) for r in ROWS})
