"""GPU: fused softmax+Dice+CE kernel vs the reference-pinned oracle and the reference's own fixtures.

Beyond the fixtures, every kernel instantiation (C = 2..16 x fp16/fp32 x channels-last/strided) and its load paths are
compared with the oracle (oracle.losses, dice_loss + cross_entropy) evaluated in fp64 on the device, on the same
fp16-rounded logits the kernel reads.  The channels-last kernel loads 8-byte words (fp16, C % 4 == 0), __half2 (fp16,
even C) or float4 (fp32, C % 4 == 0) when the base pointer is 16-byte aligned and the batch stride C*V is a multiple
of 8 elements, and one element at a time otherwise.  Bars:
  * loss, CE and Dice of the stats buffer: relative 1e-5; per-class alpha and dice: absolute 1e-5;
  * dlogits (max-norm, util.rel_err): 1e-4 in fp32, 2e-3 in fp16 (one rounding of the stored gradient).
"""
import re

import pytest
import torch

from oracle import losses as olosses
from util import launched_kernels, load_golden, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["loss_a", "loss_b", "loss_c"])
@pytest.mark.parametrize("layout", ["ncdhw", "channels_last"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("label_dtype", [torch.int64, torch.uint8])
def test_dice_ce_matches_reference_fixture(name, layout, dtype, label_dtype):
    import b200seg
    g = load_golden(name)
    xh = g["x"].to(dtype)
    x = xh.cuda()
    if layout == "channels_last":
        x = x.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)
    x.requires_grad_(True)
    y = g["y"].to(label_dtype).cuda()
    crit = b200seg.DiceCELoss(weight=g["w"])
    loss = crit(x, y)
    loss.backward()
    # oracle on the SAME (possibly fp16-rounded) logits
    xo = xh.float().requires_grad_(True)
    lo = olosses.dice_loss(xo, g["y"]) + olosses.cross_entropy(xo, g["y"], g["w"])
    lo.backward()
    assert abs(loss.item() - lo.item()) < 2e-5
    tol = 1e-4 if dtype == torch.float32 else 2e-3     # fp16: dlogits are stored in fp16
    assert rel_err(x.grad.float(), xo.grad) < tol
    if dtype == torch.float32:
        assert abs(loss.item() - (g["dice"] + g["ce"])) < 2e-5        # the reference's own numbers
        assert rel_err(x.grad, g["grad"]) < 1e-4
    # DiceLoss-compatible shim alone
    d = b200seg.DiceLoss()(x.detach(), y)
    assert abs(d.item() - olosses.dice_loss(xh.float(), g["y"]).item()) < 2e-5


def test_dice_ce_full_size_properties():
    """BASELINE size (128^3, 4 classes, fp16 NDHWC): size-independent properties of the gradient."""
    import b200seg
    torch.manual_seed(0)
    B, C, D = 1, 4, 128
    x = (torch.randn(B, D, D, D, C, device="cuda") * 2).half().permute(0, 4, 1, 2, 3).requires_grad_(True)
    y = torch.randint(0, C, (B, 1, D, D, D), device="cuda")
    w = torch.tensor([0.5, 1, 1, 1])
    loss = b200seg.DiceCELoss(weight=w)(x, y)
    # fp16 dlogits of a 2M-voxel mean are ~5e-7 (fp16 subnormals) without loss scaling — exactly why the
    # trainer uses GradScaler; check the properties at a realistic scale (device-scalar upstream grad)
    (loss * 4096.0).backward()
    assert torch.isfinite(loss)
    g = x.grad.float() / 4096.0
    # softmax-Jacobian property: gradients of one voxel sum to zero over classes
    assert g.sum(1).abs().max().item() < 2e-2 * g.abs().max().item()
    # scaling the upstream gradient scales the result linearly (GradScaler path)
    x2 = x.detach().clone().requires_grad_(True)
    (b200seg.DiceCELoss(weight=w)(x2, y) * 1024.0).backward()
    assert rel_err(x2.grad.float() / 1024.0, g) < 5e-3
    # a chunk of the volume against the oracle
    xo = x.detach().float().cpu().requires_grad_(True)
    lo = olosses.dice_loss(xo, y.cpu()) + olosses.cross_entropy(xo, y.cpu(), w)
    assert abs(lo.item() - loss.item()) < 1e-4


# ----------------------------------------------------------------------------- fp64 oracle on the device
def storage(x, layout):
    """(leaf tensor the kernel's logits are a view of, function giving that NCDHW view) for logits x [B, C, ...]:
    "ncdhw" contiguous, "channels_last" a permuted NDHWC tensor, "offset1" the same one element into its storage
    (a base pointer that is not 16-byte aligned)."""
    if layout == "ncdhw":
        return x.contiguous(), lambda t: t
    cl = x.permute(0, *range(2, x.dim()), 1).contiguous()
    to_nc = lambda t: t.permute(0, t.dim() - 1, *range(1, t.dim() - 1))      # noqa: E731
    if layout == "channels_last":
        return cl, to_nc
    assert layout == "offset1"
    flat = torch.cat([torch.zeros(1, dtype=x.dtype, device=x.device), cl.flatten()])
    return flat, lambda t: to_nc(t[1:].view(cl.shape))


def run_kernel(base, view, y, weight=None, ce_scale=1.0, dice_scale=1.0, upstream=1.0):
    """DiceCELoss on view(base); returns (loss, stats buffer, dlogits as an NCDHW view)."""
    import b200seg
    from b200seg.ops import DiceCEFn
    base = base.detach().clone().requires_grad_(True)
    loss = b200seg.DiceCELoss(weight=weight, ce_scale=ce_scale, dice_scale=dice_scale)(view(base), y)
    stats = DiceCEFn.last_stats.clone()
    (loss * upstream).backward()
    return loss.detach(), stats, view(base.grad)


def run_oracle(x, y, weight=None, ce_scale=1.0, dice_scale=1.0, upstream=1.0):
    """fp64 oracle on the device: loss, CE, Dice loss, per-class (unclamped alpha, alpha, dice) and dlogits."""
    C = x.shape[1]
    xo = x.detach().double().requires_grad_(True)
    yo = y.long()
    a_raw, alpha, dice_c = olosses.dice_terms(xo, yo)
    dl = (1 - dice_c).sum() / C
    ce = olosses.cross_entropy(xo, yo, None if weight is None else weight.to(xo.device))
    loss = ce_scale * ce + dice_scale * dl
    (loss * upstream).backward()
    return dict(loss=loss.detach(), ce=ce.detach(), dice=dl.detach(), alpha_raw=a_raw.detach(),
                alpha=alpha.detach(), dice_c=dice_c.detach(), grad=xo.grad)


def check_against_oracle(x, y, layout, weight=None, ce_scale=1.0, dice_scale=1.0, upstream=1.0):
    """x [B, C, ...] logits in their kernel dtype (fp16 values are what both sides see); returns the oracle dict."""
    C = x.shape[1]
    base, view = storage(x, layout)
    loss, st, grad = run_kernel(base, view, y, weight, ce_scale, dice_scale, upstream)
    o = run_oracle(x, y, weight, ce_scale, dice_scale, upstream)
    rel = lambda a, b: abs(float(a) - float(b)) / abs(float(b))      # noqa: E731
    assert rel(loss, o["loss"]) < 1e-5, (loss.item(), o["loss"].item())
    assert rel(st[1], o["ce"]) < 1e-5, (st[1].item(), o["ce"].item())
    assert rel(st[2], o["dice"]) < 1e-5, (st[2].item(), o["dice"].item())
    alpha, dice_c = st[4 + 2 * C:4 + 3 * C].double(), st[4 + 3 * C:4 + 4 * C].double()
    assert (alpha - o["alpha"]).abs().max().item() < 1e-5, (alpha, o["alpha"])
    assert (dice_c - o["dice_c"]).abs().max().item() < 1e-5, (dice_c, o["dice_c"])
    assert grad.dtype == x.dtype
    tol = 1e-4 if x.dtype == torch.float32 else 2e-3
    assert rel_err(grad, o["grad"]) < tol
    return o


def logits_labels(B, C, spatial, dtype, seed, background=None, label_dtype=torch.int64):
    """Random logits leaning towards the label (so Dice is neither 0 nor 1) and labels, optionally ~`background`
    of them class 0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if background is None:
        y = torch.randint(0, C, (B, 1, *spatial), generator=g, device="cuda")
    else:
        fg = torch.randint(1, C, (B, 1, *spatial), generator=g, device="cuda")
        y = torch.where(torch.rand(B, 1, *spatial, generator=g, device="cuda") < background, 0, fg)
    x = torch.randn(B, C, *spatial, generator=g, device="cuda") * 2
    x = x + 2.0 * torch.zeros_like(x).scatter_(1, y, 1.0)
    return x.to(dtype), y.to(label_dtype)


def class_weights(C, seed=0):
    return 0.5 + torch.rand(C, generator=torch.Generator().manual_seed(seed))


# ----------------------------------------------------------------------------- every instantiation
SHAPES = {"v8": (6, 8, 10), "odd": (5, 7, 9)}      # V % 8 == 0 / odd V (batch stride C*V % 8 != 0 unless 8 | C)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("label_dtype", [torch.int64, torch.uint8])
@pytest.mark.parametrize("layout", ["ncdhw", "channels_last"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", range(2, 17))
def test_dice_ce_every_instantiation(C, dtype, layout, label_dtype, shape):
    x, y = logits_labels(2, C, SHAPES[shape], dtype, seed=C, label_dtype=label_dtype)
    check_against_oracle(x, y, layout, weight=class_weights(C))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", [3, 4, 8, 14, 16])
def test_dice_ce_misaligned_channels_last(C, dtype):
    """channels-last logits one element into their storage: same strides, scalar loads and stores"""
    x, y = logits_labels(2, C, SHAPES["v8"], dtype, seed=100 + C)
    check_against_oracle(x, y, "offset1", weight=class_weights(C))


_KERNEL = re.compile(r"dice_ce_(fwd|bwd)_kernel(?:<\s*(__half|float)\s*,\s*(\d+)\s*,\s*(true|false)\s*>"
                     r"|I(6__half|f)Li(\d+)ELb([01])E)")


VECTOR_PATH_CASES = [(dtype, C, shape, layout)
                     for dtype, C in [(torch.float16, 4), (torch.float16, 14), (torch.float16, 16), (torch.float32, 4)]
                     for shape in SHAPES for layout in ["channels_last", "ncdhw", "offset1"]]


def run_vector_path_cases():
    for dtype, C, shape, layout in VECTOR_PATH_CASES:
        x, y = logits_labels(2, C, SHAPES[shape], dtype, seed=C)
        run_kernel(*storage(x, layout), y)


def test_dice_ce_vector_paths_launch():
    """The matrix above reaches both kernel variants: the channels-last one (CL = true) for aligned channels-last
    logits with C*V % 8 == 0, the strided one otherwise."""
    expected = set()
    for dtype, C, shape, layout in VECTOR_PATH_CASES:
        V = SHAPES[shape][0] * SHAPES[shape][1] * SHAPES[shape][2]
        key = ("__half" if dtype == torch.float16 else "float", C, layout == "channels_last" and (C * V) % 8 == 0)
        expected |= {("fwd", key), ("bwd", key)}
    assert {key[2] for _, key in expected} == {True, False}
    seen = set()
    for name in launched_kernels("test_gpu_loss", "run_vector_path_cases"):
        m = _KERNEL.search(name)
        if m:
            g = m.groups()
            if g[1] is not None:
                seen.add((g[0], (g[1], int(g[2]), g[3] == "true")))
            else:
                seen.add((g[0], ("__half" if g[4] == "6__half" else "float", int(g[5]), g[6] == "1")))
    assert seen, "the profiler recorded no dice_ce kernel launch"
    assert seen == expected, (sorted(expected - seen), sorted(seen - expected))


# ----------------------------------------------------------------------------- regimes
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_dice_ce_alpha_regimes(dtype):
    """One class per regime of alpha = clamp(FP / (FP + FN + s), 0.2, 0.8), each well clear of the clamp edges:
    0 under-predicted (clamped at 0.2), 1 over-predicted (clamped at 0.8), 2 inside the range, 3 absent from the labels
    (FN = 0), 4 present but never predicted (FP ~ 0)."""
    C, spatial = 5, (6, 8, 10)
    g = torch.Generator(device="cuda").manual_seed(7)
    y = torch.tensor([0, 1, 2, 4], device="cuda")[torch.randint(0, 4, (2, 1, *spatial), generator=g, device="cuda")]
    x = torch.randn(2, C, *spatial, generator=g, device="cuda")
    x = x + 2.0 * torch.zeros_like(x).scatter_(1, y, 1.0)
    x = x + torch.tensor([-2.5, 2.5, 1.0, 0.0, -40.0], device="cuda").view(1, C, 1, 1, 1)
    x = x.to(dtype)
    o = check_against_oracle(x, y, "channels_last", weight=class_weights(C))
    a = o["alpha_raw"].tolist()
    assert a[0] < 0.1 and a[1] > 0.9 and 0.3 < a[2] < 0.7 and a[3] > 0.99 and a[4] < 1e-3, a


@pytest.mark.parametrize("layout", ["ncdhw", "channels_last"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_dice_ce_confident_mistakes(dtype, layout):
    """Voxels whose labelled logit lies 80, 1 000 and 30 000 below the largest: the cross-entropy of each is its full
    log-sum-exp gap, as in F.cross_entropy, not the -log of an underflowed probability."""
    C, spatial = 4, (6, 8, 10)
    x, y = logits_labels(2, C, spatial, torch.float32, seed=11)
    xf, yf = x.flatten(2), y.flatten(2)          # views
    for j, gap in enumerate([80.0, 1000.0, 30000.0, 30000.0, 1000.0, 80.0]):
        b, v = j % 2, 17 * j + 3
        xf[b, :, v] = 5.0
        xf[b, yf[b, 0, v], v] = 5.0 - gap
    x = x.to(dtype)
    o = check_against_oracle(x, y, layout, weight=class_weights(C))
    assert o["ce"].item() > 20.0          # the six gaps dominate the mean over 960 voxels


@pytest.mark.parametrize("upstream", [65536.0, 0.5])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("weighted", [True, False])
def test_dice_ce_scales_and_upstream(weighted, dtype, upstream):
    C = 6
    x, y = logits_labels(2, C, (6, 8, 10), dtype, seed=21)
    check_against_oracle(x, y, "channels_last", weight=class_weights(C) if weighted else None, ce_scale=0.5,
                         dice_scale=2.0, upstream=upstream)


@pytest.mark.parametrize("C", [1, 17])
def test_dice_ce_class_count_out_of_range(C):
    import b200seg
    x, y = logits_labels(1, max(C, 2), (4, 4, 4), torch.float16, seed=0)
    x = x[:, :C].contiguous() if C == 1 else x
    y = y.clamp_max(C - 1)
    with pytest.raises(b200seg.B200SegError):
        b200seg.DiceCELoss()(x, y)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------- benchmark shapes
def _bench_weight(workload):
    import bench
    return torch.tensor(bench.WORKLOADS[workload][3], dtype=torch.float32)


@pytest.mark.parametrize("workload,B,C,spatial", [
    ("resunet_acdc_128", 1, 4, (128, 128, 128)),
    ("resunet_kits_160", 2, 3, (160, 160, 80)),
    ("medformer_bcv_96", 1, 14, (96, 96, 96)),
    ("swin_unetr_amos_128", 1, 16, (128, 128, 128)),
])
def test_dice_ce_benchmark_shapes(workload, B, C, spatial):
    """fp16 channels-last logits at each benchmark's head, ~70 % background, GradScaler's initial upstream gradient"""
    w = _bench_weight(workload)
    assert w.numel() == C
    x, y = logits_labels(B, C, spatial, torch.float16, seed=C, background=0.7)
    check_against_oracle(x, y, "channels_last", weight=w, upstream=65536.0)


def test_dice_ce_medformer_aux_view():
    """MedFormer's auxiliary head: channels 0..13 of a 16-channel channels-last buffer (DiceCEFn copies it to NCDHW)"""
    C, spatial = 14, (96, 96, 96)
    w = _bench_weight("medformer_bcv_96")
    x, y = logits_labels(1, 16, spatial, torch.float16, seed=5, background=0.7)
    y = y.clamp_max(C - 1)
    buf = x.permute(0, 2, 3, 4, 1).contiguous()
    view = lambda t: t[..., :C].permute(0, 4, 1, 2, 3)      # noqa: E731
    loss, st, grad = run_kernel(buf, view, y, w, upstream=65536.0)
    o = run_oracle(view(buf), y, w, upstream=65536.0)
    assert abs(loss.item() - o["loss"].item()) < 1e-5 * o["loss"].item()
    assert (st[4 + 2 * C:4 + 3 * C].double() - o["alpha"]).abs().max().item() < 1e-5
    assert (st[4 + 3 * C:4 + 4 * C].double() - o["dice_c"]).abs().max().item() < 1e-5
    assert rel_err(grad, o["grad"]) < 2e-3
