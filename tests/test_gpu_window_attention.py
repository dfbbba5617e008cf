"""GPU: the SwinUNETR window-attention kernels (csrc/swin_mma.cu on the tensor cores, csrc/swin.cu on the CUDA cores,
geometry in csrc/swin_geom.cuh) against oracle.swin_ops.window_attention_core in float64 — the operator restated from
the reference's pinned pieces and itself tied to the reference-made block fixtures (tests/test_swin_host.py).

  * the operator matrix: every window geometry that reaches a different branch of the index arithmetic (padding, shift
    mask, windows clamped by `<=`, D = 1, n = 1, n = 352, non-cubic windows, large logits), on the three kernel
    families (fp16 tensor-core, fp16 CUDA-core, fp32 CUDA-core) and every head size each one serves, plus the
    training-stage shapes of the benchmarked SwinUNETR (feature_size 48, 128^3: 64^3 / 32^3 / 16^3 with 3 / 6 / 12
    heads of 16);
  * which kernels each call launches, a forward and a backward on different paths, the ABI's overwrite / `+=`
    contract, the refusal of windows larger than a CTA, and run-to-run reproducibility;
  * the benchmarked SwinUNETR configuration end to end (AMP step against the fp32 oracle, two identical TrainSteps).

Every comparison is a max-norm error relative to the reference tensor's own max (dq, dk and dv separately, so an error
in dq cannot hide behind a larger dv).  fp16 rows compare with the reference rounded where the reference's autocast
rounds (bias, q * scale, probabilities)."""
import ctypes
import json
import os
import types

import pytest
import torch

from oracle import losses as olosses
from oracle import swin_ops as so
from oracle import swin_unetr as osw
from oracle import unet3d as ounet
from oracle.synth import make_volume
from util import global_l2, launched_kernels_each, rel_err

pytestmark = pytest.mark.gpu

# Bars set from the largest error measured over this file on an H100 80GB HBM3 (SXM, 700 W power limit), with at most
# 3x headroom (DESIGN.md §4 lists the rows that set them):
#            out                      dq / dk / dv             dtable, dbias
#   fp32     2.4e-6 large_logit        3.0e-6 large_logit       4.8e-6 stage 32^3 dbias_v
#   fp16     2.0e-3 large_logit cc16   3.2e-3 large_logit cc16  1.6e-3 pad_bias8 dbias_k
# The fp16 CUDA-core kernels keep q * scale and the probabilities in fp32 where the reference (and the tensor-core
# kernels) round them to fp16, so against the rounded reference they set the fp16 maxima (the tensor-core rows stay
# below 6.3e-4 / 1.8e-3 / 1.6e-3).
BARS = {"fp32": (6e-6, 8e-6, 1.2e-5),
        "fp16": (4e-3, 8e-3, 4e-3)}

# id: dims, window, shift, extra (qkv scale, table scale, bias centre); B = 2 unless a row says otherwise
GEOM = {
    "exact": ((14, 14, 14), (7, 7, 7), (0, 0, 0)),                 # no padding, no mask
    "exact_shift": ((14, 14, 14), (7, 7, 7), (3, 3, 3)),           # mask, no padding
    "pad": ((9, 10, 11), (7, 7, 7), (0, 0, 0)),                    # padding on every axis
    "pad_shift": ((16, 16, 16), (7, 7, 7), (3, 3, 3)),             # stage-3 geometry of a 128^3 input (P = 21)
    "clamp_w": ((9, 14, 5), (7, 7, 7), (3, 3, 3)),                 # W clamped, its shift dropped; D / H shifted + padded
    "eq_window": ((7, 14, 12), (7, 7, 7), (3, 3, 3)),              # a dim equal to the window clamps (`<=`)
    "clamp_all": ((4, 6, 5), (7, 7, 7), (3, 3, 3)),                # all clamped, unmasked, index decoded in 7^3
    "thin": ((1, 12, 12), (7, 7, 7), (3, 3, 3)),                   # D = 1, n = 49 (NP = 64)
    "single": ((1, 1, 1), (7, 7, 7), (3, 3, 3)),                   # n = 1
    "small_win": ((8, 9, 10), (4, 4, 4), (2, 0, 2)),               # non-7 window, partial shift
    "aniso": ((6, 11, 16), (3, 5, 7), (1, 2, 3)),                  # distinct strides in L_i - L_j + K0
    "n_max": ((16, 11, 8), (8, 11, 4), (4, 0, 2)),                 # n = 352 = one token per thread, no padded keys
    "large_logit": ((14, 14, 14), (7, 7, 7), (3, 3, 3)),           # qkv x4, table x3: running max moves between key blocks
    "pad_bias8": ((9, 10, 11), (7, 7, 7), (3, 3, 3)),              # padding with a qkv bias of magnitude ~8 (not fp16-exact)
}
EXTRA = {"large_logit": dict(qscale=3.2, tscale=1.5), "pad_bias8": dict(bcentre=8.0)}

PATHS = {"mma": (torch.float16, "1"), "cc16": (torch.float16, "0"), "fp32": (torch.float32, "1")}


def _err(a, b):
    """max |a - b| over max |b|; absolute where b is exactly zero (the dq, dk and d(table) of a one-token window: its
    probability is 1 whatever the score).  The inputs are of unit scale."""
    a, b = a.detach().double(), b.detach().double()
    scale = b.abs().max().item()
    return (a - b).abs().max().item() / (scale if scale > 0 else 1.0)


def _inputs(dims, window, heads, dh, B, seed, qscale=0.8, tscale=0.5, bscale=0.3, bcentre=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = heads * dh
    T = (2 * window[0] - 1) * (2 * window[1] - 1) * (2 * window[2] - 1)
    qkv = torch.randn(B, *dims, 3 * C, generator=g, device="cuda") * qscale
    bias = torch.randn(3 * C, generator=g, device="cuda") * bscale
    bias = bias + bcentre * torch.sign(bias)
    table = torch.randn(T, heads, generator=g, device="cuda") * tscale
    dout = torch.randn(B, *dims, C, generator=g, device="cuda")
    return qkv, bias, table, dout


def _reference(qkv, bias, table, dout, heads, window, shift, fp16):
    """window_attention_core in float64 on the kernel's (rounded) inputs: out, dqkv, dtable, dbias (dbias None without
    a bias)."""
    x = qkv.double().requires_grad_(True)
    b = None if bias is None else bias.double().requires_grad_(True)
    t = table.double().requires_grad_(True)
    y = so.window_attention_core(x, b, t, heads, window, shift, fp16_rounding=fp16)
    y.backward(dout.double())
    return y.detach(), x.grad, t.grad, None if b is None else b.grad


def _compare(tag, got, ref, C, padded, fp16):
    """got / ref: (out, dqkv, dtable, dbias).  Returns the error per quantity after checking the bars."""
    out, dqkv, dtable, dbias = got
    rout, rdqkv, rdtable, rdbias = ref
    errs = {"out": _err(out, rout), "dtable": _err(dtable, rdtable)}
    for i, nm in enumerate(("dq", "dk", "dv")):
        errs[nm] = _err(dqkv[..., i * C:(i + 1) * C], rdqkv[..., i * C:(i + 1) * C])
    if dbias is not None:
        assert torch.count_nonzero(dbias[:C]) == 0, "padding queries carry no gradient: the q third of dbias is zero"
        if padded:
            errs["dbias_k"] = _err(dbias[C:2 * C], rdbias[C:2 * C])
            errs["dbias_v"] = _err(dbias[2 * C:], rdbias[2 * C:])
        else:
            assert torch.count_nonzero(dbias) == 0, "no padding token, no gradient into the qkv bias"
    print("WINATTN_ERR %s %s" % (tag, json.dumps({k: float("%.3e" % v) for k, v in errs.items()})))
    b_out, b_g, b_p = BARS["fp16" if fp16 else "fp32"]
    assert errs["out"] < b_out, errs
    assert max(errs[k] for k in ("dq", "dk", "dv")) < b_g, errs
    assert max(v for k, v in errs.items() if k.startswith("dtable") or k.startswith("dbias")) < b_p, errs
    return errs


def _check(monkeypatch, tag, geom, heads, dh, path, B=2, bias=True, seed=0, chunk=64, **extra):
    from b200seg.swin_unetr import WindowAttnFn
    dims, window, shift = geom
    dtype, mma = PATHS[path]
    monkeypatch.setenv("B200SEG_WINATTN_MMA", mma)
    qkv, qb, table, dout = _inputs(dims, window, heads, dh, B, seed, **extra)
    qkv, dout = qkv.to(dtype), dout.to(dtype)
    x = qkv.clone().requires_grad_(True)
    b = qb.clone().requires_grad_(True) if bias else None
    t = table.clone().requires_grad_(True)
    y = WindowAttnFn.apply(x, b, t, heads, window, shift)
    y.backward(dout)
    got = (y.detach(), x.grad, t.grad, None if b is None else b.grad)
    del x, y
    ref = _reference(qkv, qb if bias else None, table, dout, heads, window, shift, dtype == torch.float16)
    ws, _ = so.get_window_size(dims, window, shift)
    padded = any(d % w for d, w in zip(dims, ws))
    return _compare(tag, got, ref, heads * dh, padded, dtype == torch.float16)


# ----------------------------------------------------------------------------------------------- the operator matrix
MATRIX = [(row, path, dh) for row in GEOM for path in ("mma", "cc16", "fp32") for dh in (8, 16, 32)]
MATRIX += [(row, "cc16", dh) for row in ("pad_shift", "clamp_w", "aniso", "n_max", "pad_bias8") for dh in (4, 12, 24)]


@pytest.mark.parametrize("row,path,dh", MATRIX, ids=["%s-%s-dh%d" % m for m in MATRIX])
def test_operator_matrix(monkeypatch, row, path, dh):
    """fp16 dh 8 / 16 / 32 run on the tensor cores (mma) or, forced, on the CUDA cores (cc16); fp16 dh 4 / 12 / 24 only
    have the CUDA-core kernel; fp32 always runs on the CUDA cores."""
    i = list(GEOM).index(row)
    heads = 2 + (i + dh // 8) % 2
    _check(monkeypatch, "%s-%s-dh%d" % (row, path, dh), GEOM[row], heads, dh, path, seed=100 * i + dh, **EXTRA.get(row, {}))


@pytest.mark.parametrize("path", ["mma", "cc16", "fp32"])
def test_twelve_heads(monkeypatch, path):
    """heads = 12 of 16 (stage 3 of SwinUNETR at feature_size 48) on the padded, shifted stage-3 geometry."""
    _check(monkeypatch, "heads12-" + path, GEOM["pad_shift"], 12, 16, path, seed=7)


@pytest.mark.parametrize("path", ["mma", "cc16", "fp32"])
def test_no_qkv_bias(monkeypatch, path):
    """qkv_bias=None: a padding token's q / k / v is zero and nothing is accumulated into a bias."""
    _check(monkeypatch, "nobias-" + path, GEOM["pad_shift"], 3, 16, path, bias=False, seed=8)


# (dims, heads, B, path): the bench configuration's attention shapes (feature_size 48, dh 16, window 7)
STAGES = [((64, 64, 64), 3, 1, "mma"), ((32, 32, 32), 6, 1, "mma"), ((16, 16, 16), 12, 1, "mma"),
          ((32, 32, 32), 6, 2, "mma"), ((32, 32, 32), 6, 1, "fp32")]


@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("dims,heads,B,path", STAGES, ids=["%d-h%d-B%d-%s" % (s[0][0], s[1], s[2], s[3]) for s in STAGES])
def test_training_stage_shapes(monkeypatch, dims, heads, B, path, shift):
    _check(monkeypatch, "stage%d-h%d-B%d-%s-s%d" % (dims[0], heads, B, path, shift), (dims, (7, 7, 7), (shift,) * 3),
           heads, 16, path, B=B, seed=dims[0] + heads + B + shift)


# ----------------------------------------------------------------------------------------------- the raw ABI
def _raw(qkv, bias, table, dout, heads, window, shift, out=None, dqkv=None, dtable=None, dbias=None):
    """b200seg_window_attn_fwd then _bwd on caller-owned buffers (WindowAttnFn allocates its own)."""
    from b200seg import _lib
    from b200seg.ops import _dt, _stream
    B, D, H, W, C3 = qkv.shape
    dh = C3 // 3 // heads
    win, sft = (ctypes.c_int * 3)(*window), (ctypes.c_int * 3)(*shift)
    lse = torch.empty(_lib.load().b200seg_window_attn_workspace(B, D, H, W, heads, win) // 4, device="cuda")
    delta = torch.empty_like(lse)
    out = torch.empty(B, D, H, W, C3 // 3, dtype=qkv.dtype, device="cuda") if out is None else out
    dqkv = torch.empty_like(qkv) if dqkv is None else dqkv
    dtable = torch.zeros_like(table) if dtable is None else dtable
    dbias = torch.zeros_like(bias) if dbias is None else dbias
    _lib.call("b200seg_window_attn_fwd", qkv.data_ptr(), bias.data_ptr(), table.data_ptr(), out.data_ptr(), lse.data_ptr(),
              B, D, H, W, heads, dh, win, sft, _dt(qkv), _stream())
    _lib.call("b200seg_window_attn_bwd", qkv.data_ptr(), bias.data_ptr(), table.data_ptr(), out.data_ptr(), dout.data_ptr(),
              lse.data_ptr(), delta.data_ptr(), dqkv.data_ptr(), dtable.data_ptr(), dbias.data_ptr(), B, D, H, W, heads, dh,
              win, sft, _dt(qkv), _stream())
    return out, dqkv, dtable, dbias


def _misaligned(t):
    """t's values in a contiguous view whose address is 8 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 8, dtype=t.dtype, device=t.device)
    v = buf[8 // t.element_size():8 // t.element_size() + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 8
    return v


ROUTING_CASES = ["dh8", "dh16", "dh32", "dh4", "dh12", "dh24", "misaligned", "forced"]
MIXED_ROWS = ["pad_shift", "clamp_w", "large_logit"]
_NAMES = {}


def _kernels(fn, arg):
    """names of the window-attention kernels fn(arg) (_routing_launch or _mixed_launch) launches.  They are recorded by
    the profiler in a fresh process, all cases in one: a profiling session late in a long pytest process was seen to
    keep only the last kernel."""
    if not _NAMES:
        calls = [("_routing_launch", (c,)) for c in ROUTING_CASES] + [("_mixed_launch", (r,)) for r in MIXED_ROWS]
        for call, names in zip(calls, launched_kernels_each("test_gpu_window_attention", calls)):
            _NAMES[call] = sorted({n for n in names if "win_attn" in n})
    return _NAMES[(fn, (arg,))]


def _routing_inputs(case):
    dh = int(case[2:]) if case.startswith("dh") else 16
    dims, window, shift = GEOM["pad_shift"]
    qkv, qb, table, dout = _inputs(dims, window, 3, dh, 2, seed=dh)
    qkv, dout = qkv.half(), dout.half()
    return dh, (window, shift), (qkv, qb, table, dout)


def _routing_launch(case):
    os.environ["B200SEG_WINATTN_MMA"] = "0" if case == "forced" else "1"      # a process of its own: no restore
    _, (window, shift), (qkv, qb, table, dout) = _routing_inputs(case)
    x = _misaligned(qkv) if case == "misaligned" else qkv
    _raw(x, qb, table, dout, 3, window, shift)


def _mixed_inputs(row):
    dims, window, shift = GEOM[row]
    qkv, qb, table, dout = _inputs(dims, window, 3, 16, 2, seed=31, **EXTRA.get(row, {}))
    return (window, shift), (qkv.half(), qb, table, dout.half())


def _mixed_launch(row):
    os.environ["B200SEG_WINATTN_MMA"] = "1"
    (window, shift), (qkv, qb, table, dout) = _mixed_inputs(row)
    _raw(qkv, qb, table, _misaligned(dout), 3, window, shift)


MMA_NAMES = ("win_attn_fwd_mma_kernel<%d>", "win_attn_bwd_q_mma_kernel<%d>", "win_attn_bwd_kv_mma_kernel<%d>")
CC_NAMES = ("win_attn_fwd_kernel<__half>", "win_attn_bwd_q_kernel<__half>", "win_attn_bwd_kv_kernel<__half>")


@pytest.mark.parametrize("case", ROUTING_CASES)
def test_kernel_routing(monkeypatch, case):
    """fp16 with dh 8 / 16 / 32 launches the tensor-core forward and both tensor-core backward passes; dh 4 / 12 / 24, a
    qkv that is not 16-byte aligned and B200SEG_WINATTN_MMA=0 launch the CUDA-core kernels (and still compute the
    operator)."""
    monkeypatch.setenv("B200SEG_WINATTN_MMA", "0" if case == "forced" else "1")
    dh, (window, shift), (qkv, qb, table, dout) = _routing_inputs(case)
    x = _misaligned(qkv) if case == "misaligned" else qkv
    # the raw entry points with fresh outputs, as WindowAttnFn calls them (dqkv is a new, aligned tensor)
    names = _kernels("_routing_launch", case)
    res = {"r": _raw(x, qb, table, dout, 3, window, shift)}
    print(case, names)
    expect = [n % dh for n in MMA_NAMES] if case in ("dh8", "dh16", "dh32") else list(CC_NAMES)
    for e in expect:
        assert sum(e in n for n in names) == 1, (e, names)
    assert len(names) == 3, names
    ref = _reference(qkv, qb, table, dout, 3, window, shift, True)
    assert _err(res["r"][0], ref[0]) < BARS["fp16"][0]
    assert _err(res["r"][1], ref[1]) < BARS["fp16"][1]


@pytest.mark.parametrize("row", MIXED_ROWS)
def test_mixed_paths(monkeypatch, row):
    """A dout that is not 16-byte aligned sends the backward to the CUDA cores after a tensor-core forward: the CUDA-core
    passes recompute P with an fp32 q * scale from an lse the tensor-core forward made with an fp16 one.  The result
    still meets the fp16 bars."""
    monkeypatch.setenv("B200SEG_WINATTN_MMA", "1")
    (window, shift), (qkv, qb, table, dout) = _mixed_inputs(row)
    names = _kernels("_mixed_launch", row)
    res = {"r": _raw(qkv, qb, table, _misaligned(dout), 3, window, shift)}
    assert len(names) == 3, names
    for e in (MMA_NAMES[0] % 16, CC_NAMES[1], CC_NAMES[2]):
        assert sum(e in n for n in names) == 1, (e, names)
    ref = _reference(qkv, qb, table, dout, 3, window, shift, True)
    _compare("mixed-" + row, res["r"], ref, 48, True, True)


@pytest.mark.parametrize("path", ["mma", "cc16", "fp32"])
@pytest.mark.parametrize("row", ["pad_shift", "clamp_w", "thin"])
def test_abi_overwrite_and_accumulate(monkeypatch, path, row):
    """out and dqkv prefilled with NaN: every real voxel is written (a skipped tile would leave NaN).  dtable and
    dbias_pad prefilled with random values: the ABI adds the gradient to them (`+=`)."""
    dtype, mma = PATHS[path]
    monkeypatch.setenv("B200SEG_WINATTN_MMA", mma)
    dims, window, shift = GEOM[row]
    qkv, qb, table, dout = _inputs(dims, window, 3, 16, 2, seed=41)
    qkv, dout = qkv.to(dtype), dout.to(dtype)
    g = torch.Generator(device="cuda").manual_seed(42)
    t0, b0 = torch.randn(table.shape, generator=g, device="cuda"), torch.randn(qb.shape, generator=g, device="cuda")
    out = torch.full((*qkv.shape[:-1], 48), float("nan"), dtype=dtype, device="cuda")
    dqkv = torch.full_like(qkv, float("nan"))
    out, dqkv, dtable, dbias = _raw(qkv, qb, table, dout, 3, window, shift, out, dqkv, t0.clone(), b0.clone())
    assert not torch.isnan(out).any() and not torch.isnan(dqkv).any()
    ref = _reference(qkv, qb, table, dout, 3, window, shift, dtype == torch.float16)
    _compare("abi-%s-%s" % (row, path), (out, dqkv, dtable - t0, dbias - b0), ref, 48, True, dtype == torch.float16)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_window_larger_than_a_cta_is_refused(dtype):
    """n = 7 * 7 * 8 = 392 tokens > 352 (one token per thread): an error, not a truncated window."""
    from b200seg._lib import B200SegError
    from b200seg.swin_unetr import WindowAttnFn
    qkv = torch.zeros(1, 8, 8, 9, 3 * 32, dtype=dtype, device="cuda")
    table = torch.zeros(13 * 13 * 15, 2, device="cuda")
    with pytest.raises(B200SegError):
        WindowAttnFn.apply(qkv, None, table, 2, (7, 7, 8), (0, 0, 0))


@pytest.mark.parametrize("path", ["mma", "cc16", "fp32"])
def test_reproducible(monkeypatch, path):
    """Two identical calls: out and dqkv bit-identical; dtable and dbias are sums of fp32 atomics (DESIGN §4a), so only
    their rounding may differ."""
    dtype, mma = PATHS[path]
    monkeypatch.setenv("B200SEG_WINATTN_MMA", mma)
    dims, window, shift = GEOM["pad_shift"]
    qkv, qb, table, dout = _inputs(dims, window, 3, 16, 2, seed=51)
    qkv, dout = qkv.to(dtype), dout.to(dtype)
    a = _raw(qkv, qb, table, dout, 3, window, shift)
    b = _raw(qkv, qb, table, dout, 3, window, shift)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    # each dbias element sums ~10^4 padding keys' dk / dv: 1.0e-6 measured (fp32), the order of those adds is free
    assert _err(a[2], b[2]) < 3e-6 and _err(a[3], b[3]) < 3e-6


# ----------------------------------------------------------------------------------------------- the bench configuration
AMOS = dict(dimension="3d", model="swin_unetr", in_chan=1, classes=16, window_size=[128, 128, 128], base_chan=48)


def _seeded_state(shapes):
    sd = ounet.make_state_dict(shapes, seed=7)
    for k in sd:
        if k.endswith("norm1.weight") or k.endswith("norm2.weight") or k.endswith("norm.weight"):
            sd[k] = 1.0 + 0.1 * sd[k] / sd[k].abs().max()
        if k.endswith("relative_position_bias_table"):
            sd[k] = sd[k] * 3.0
    return sd


def test_fullsize_amp_step():
    """get_model's SwinUNETR as bench.py times it (128^3, feature_size 48, 16 classes, AMP): one forward / backward
    against the fp32 oracle (stock torch autocast of the same oracle is the fp16 noise floor), then two identical
    TrainSteps from the same state give the same loss and bit-identical parameters and EMA outside the parameters fed
    by float atomics."""
    import b200seg
    from b200seg.train import TrainStep
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        args = types.SimpleNamespace(**AMOS)
        sd = _seeded_state(osw.swin_unetr_param_shapes(1, 16, 48))
        img, lab = make_volume(1, 128, 128, 128, 16, seed=2025)
        img, lab = img.cuda(), lab.cuda()
        w = torch.tensor([0.5] + [1.0] * 15)

        def oracle(autocast, S):
            s = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                lo = osw.swin_unetr_forward(s, img)
                loss = olosses.total_loss(lo, lab, w.cuda())
            (loss * S).backward()
            return lo.detach().double().cpu(), loss.item(), {k: (v.grad / S).double().cpu() for k, v in s.items()}
        l32, loss32, g32 = oracle(False, 1.0)
        l_st, _, g_st = oracle(True, 1024.0)
        torch.cuda.empty_cache()

        net = b200seg.get_model(args)
        missing = net.load_state_dict(sd, strict=False)
        assert all(k.endswith("relative_position_index") for k in missing.missing_keys) and not missing.unexpected_keys
        net = net.cuda()
        S = 1024.0
        with torch.autocast("cuda", dtype=torch.float16):
            logits = net(img)
            loss = b200seg.DiceCELoss(weight=w)(logits, lab)
        (loss * S).backward()
        lg = logits.detach().double().cpu()
        ours = {k: (p.grad / S).double().cpu() for k, p in net.named_parameters()}
        assert set(ours) == set(g32)
        e, e_st = rel_err(lg, l32), rel_err(l_st, l32)
        l2, l2_st = global_l2(ours, g32), global_l2(g_st, g32)
        agree = (lg.argmax(1) == l32.argmax(1)).float().mean().item()
        print("swin_unetr amos 128 AMP: logits rel err vs fp32 oracle %.2e (stock autocast %.2e); loss %.5f (oracle "
              "%.5f); grads global-L2 %.2e (stock autocast %.2e); label agreement %.5f"
              % (e, e_st, loss.item(), loss32, l2, l2_st, agree))
        assert e < max(5e-2, 3 * e_st)
        assert abs(loss.item() - loss32) < 2e-2
        assert l2 < max(0.1, 3 * l2_st)
        assert agree > 0.97
        del net, logits, loss, ours, g32, g_st
        torch.cuda.empty_cache()

        def one_step():
            n = b200seg.get_model(args)
            n.load_state_dict(sd, strict=False)
            n = n.cuda()
            ema = b200seg.get_model(args)
            ema.load_state_dict(sd, strict=False)
            ema = ema.cuda()
            step = TrainStep(n, ema, ce_weight=w, amp=True)
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
        print("swin_unetr amos 128 TrainStep: loss %.6f / %.6f, %d of %d parameter tensors updated; differing between "
              "the two runs: %s" % (la, lb, moved, len(pa), differ))
        assert la == lb
        assert moved > len(pa) // 2

        def atomic(k):
            # win_attn_bwd_q(_mma)_kernel sums d(bias table) over windows with float atomics
            if k.endswith("attn.relative_position_bias_table"):
                return True
            # win_attn_bwd_kv(_mma)_kernel sums the padding tokens' dk / dv into d(qkv bias) with float atomics
            if k.endswith("attn.qkv.bias"):
                return True
            # the patch embedding is a 1x1x1 GEMM over 8 = 2x2x2 input channels: fewer than the tensor-core weight
            # gradient takes (Cin % 16), so conv_wgrad_direct_kernel adds its dW / dbias partials with float atomics
            if k.startswith("swinViT.patch_embed.proj."):
                return True
            # LayerNormFn's backward (b200seg_layernorm_bwd) sums d(gamma) / d(beta) with float atomics
            return ".norm" in k and k.split(".")[-1] in ("weight", "bias")
        assert all(atomic(k) for k in differ), differ
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
