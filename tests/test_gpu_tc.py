"""GPU: the wgmma implicit-GEMM conv (ALGO_TC) against the CUDA-core kernel (same rounding model) and a
PyTorch fp32 evaluation, across the mechanisms it has (K steps/chunks, tap shifts, N tiles, ragged tiles,
loader normalise+ReLU, residual / dgrad epilogues, InstanceNorm sums)."""
import pytest
import torch
import torch.nn.functional as F

from util import rel_err

pytestmark = pytest.mark.gpu

CASES = [
    # Cin, Cout, k, (B, D, H, W), mode
    (16, 16, (1, 1, 1), (1, 1, 16, 8), "plain"),
    (32, 32, (3, 3, 3), (1, 4, 16, 16), "norm"),
    (32, 64, (3, 3, 3), (2, 3, 20, 12), "norm"),
    (96, 64, (1, 3, 3), (1, 2, 32, 16), "normres"),
    (64, 128, (3, 3, 3), (1, 3, 16, 16), "normres"),
    (192, 64, (3, 3, 3), (1, 2, 16, 8), "norm"),
    (64, 320, (3, 3, 3), (1, 2, 16, 8), "norm"),
    (128, 256, (3, 3, 3), (1, 2, 16, 8), "norm"),
    (64, 32, (3, 3, 3), (2, 3, 16, 16), "dgrad"),
    (32, 32, (1, 3, 3), (1, 8, 64, 64), "normres"),
    (128, 128, (3, 3, 3), (1, 16, 64, 64), "normres"),   # many tiles per CTA, streamed weights
    (64, 64, (1, 3, 3), (1, 16, 128, 128), "normres"),   # resident weights, many tiles
    (64, 32, (3, 3, 3), (64, 1, 16, 8), "norm"),          # large B*Cin tables leave 3 A stages: 1-stage cp.async loader
]


@pytest.mark.parametrize("Cin,Cout,k,shape,mode", CASES)
def test_tc_conv_matches_direct_and_torch(Cin, Cout, k, shape, mode):
    from b200seg import ops, _lib
    B, D, H, W = shape
    torch.manual_seed(7)
    x = torch.randn(B, D, H, W, Cin, device="cuda").half()
    w = torch.randn(Cout, Cin, *k, device="cuda") * (1.0 / (Cin * k[0] * k[1] * k[2]) ** 0.5)
    st = ops.instnorm_stats(x, 0, Cin) if mode in ("norm", "normres") else None
    act = ops.ACT_RELU if st is not None else ops.ACT_NONE
    res = torch.randn(B, D, H, W, Cout, device="cuda").half() if mode == "normres" else None
    dg = None
    if mode == "dgrad":
        gx = torch.randn(B, D, H, W, Cout, device="cuda").half()
        dg = (gx, 0, ops.instnorm_stats(gx, 0, Cout), ops.ACT_RELU)
    assert ops.conv_algo(Cin, Cout, k, torch.float16, B) == _lib.ALGO_TC
    ys = {}
    for algo in (_lib.ALGO_DIRECT, _lib.ALGO_TC):
        wp = ops.pack_weight(w, torch.float16, layout=algo)
        ys[algo] = ops.conv3d_fwd(x, 0, Cin, st, act, wp, Cout, k, residual=res, dgrad_of=dg, algo=algo)
    torch.cuda.synchronize()
    (yd, sd), (yt, stt) = ys[_lib.ALGO_DIRECT], ys[_lib.ALGO_TC]
    assert rel_err(yt.float(), yd.float()) < 3e-3
    assert rel_err(stt, sd) < 1e-3
    if mode != "dgrad":
        xf = x.float().permute(0, 4, 1, 2, 3)
        a = F.relu(F.instance_norm(xf, eps=1e-4)).half().float() if st is not None else xf
        ref = F.conv3d(a, w.half().float(), padding=[i // 2 for i in k])
        if res is not None:
            ref = ref.half().float() + res.float().permute(0, 4, 1, 2, 3)
        assert rel_err(yt.float().permute(0, 4, 1, 2, 3), ref) < 4e-3


WCASES = [
    (16, 16, (1, 1, 1), (1, 1, 16, 8), False),
    (32, 32, (3, 3, 3), (1, 4, 16, 16), True),
    (32, 64, (3, 3, 3), (2, 3, 20, 12), True),
    (96, 64, (1, 3, 3), (1, 2, 32, 16), True),
    (128, 128, (3, 3, 3), (1, 4, 32, 32), True),
    (128, 128, (3, 3, 3), (1, 16, 64, 64), True),     # many voxel tiles per CTA on the 2-slot ring
    (32, 32, (1, 3, 3), (1, 16, 128, 128), True),     # 132-way split-K, long accumulation
    (192, 256, (3, 3, 3), (1, 2, 16, 16), True),
    (64, 320, (3, 3, 3), (1, 2, 16, 8), True),
]


@pytest.mark.parametrize("Cin,Cout,k,shape,normed", WCASES)
def test_tc_wgrad_matches_direct_and_torch(Cin, Cout, k, shape, normed):
    from b200seg import ops, _lib
    B, D, H, W = shape
    torch.manual_seed(9)
    x = torch.randn(B, D, H, W, Cin, device="cuda").half()
    dy = torch.randn(B, D, H, W, Cout, device="cuda").half()
    st = ops.instnorm_stats(x, 0, Cin) if normed else None
    act = ops.ACT_RELU if normed else ops.ACT_NONE
    dwd, _ = ops.conv3d_wgrad(x, 0, Cin, st, act, dy, 0, Cout, k, algo=_lib.ALGO_DIRECT)
    dwt, _ = ops.conv3d_wgrad(x, 0, Cin, st, act, dy, 0, Cout, k, algo=_lib.ALGO_TC)
    assert rel_err(dwt, dwd) < 2e-3
    xf = x.float().permute(0, 4, 1, 2, 3)
    a = (F.relu(F.instance_norm(xf, eps=1e-4)).half().float() if normed else xf)
    w = torch.zeros(Cout, Cin, *k, device="cuda", requires_grad=True)
    F.conv3d(a, w, padding=[i // 2 for i in k]).backward(dy.float().permute(0, 4, 1, 2, 3))
    assert rel_err(dwt, w.grad) < 3e-3


@pytest.mark.parametrize("Cin,Cout,k,shape", [(48, 144, (1, 1, 1), (1, 8, 16, 16)),        # qkv Linear of SwinUNETR stage 1
                                              (192, 48, (1, 1, 1), (2, 4, 16, 8)),         # fc2
                                              (768, 3072, (1, 1, 1), (1, 4, 4, 4)),        # fc1 of the last stage: > 512 output channels
                                              (32, 24, (3, 3, 3), (1, 3, 16, 16))])
def test_biased_wgrad_takes_tensor_cores(Cin, Cout, k, shape):
    """A weight gradient WITH a bias gradient (every nn.Linear of SwinUNETR) = the column-sum pass + the tensor-core kernel
    (ALGO_AUTO), against the CUDA-core kernel that computes both (ALGO_DIRECT) and PyTorch."""
    from b200seg import ops, _lib
    B, D, H, W = shape
    torch.manual_seed(13)
    x = torch.randn(B, D, H, W, Cin, device="cuda").half()
    dy = torch.randn(B, D, H, W, Cout, device="cuda").half()
    c0 = _lib.launch_count
    dwa, dba = ops.conv3d_wgrad(x, 0, Cin, None, ops.ACT_NONE, dy, 0, Cout, k, want_bias=True, algo=_lib.ALGO_AUTO)
    dwd, dbd = ops.conv3d_wgrad(x, 0, Cin, None, ops.ACT_NONE, dy, 0, Cout, k, want_bias=True, algo=_lib.ALGO_DIRECT)
    torch.cuda.synchronize()
    assert rel_err(dwa, dwd) < 2e-3 and rel_err(dba, dbd) < 2e-3
    w = torch.zeros(Cout, Cin, *k, device="cuda", requires_grad=True)
    b = torch.zeros(Cout, device="cuda", requires_grad=True)
    F.conv3d(x.float().permute(0, 4, 1, 2, 3), w, b, padding=[i // 2 for i in k]).backward(dy.float().permute(0, 4, 1, 2, 3))
    assert rel_err(dwa, w.grad) < 3e-3 and rel_err(dba, b.grad) < 1e-3
    assert not torch.equal(dwa, dwd)           # different kernels (split-K order), not the same code path twice
