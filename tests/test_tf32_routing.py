"""CPU: the TF32 selection rule of the fp32 convolutions (ops.conv_algo, b200seg_conv3d_algo_tf32) and the repacking of a
PackedWeights holder when the rule's answer changes.

fp32 convolutions run on the TF32 tensor cores only while torch allows TF32 matmuls
(torch.backends.cuda.matmul.fp32_precision == 'tf32'); at the default ('none', or 'ieee' after a reset) every fp32 shape
stays on the exact CUDA-core path.  cuDNN's conv flag, which defaults to 'tf32', is not followed."""
import os

import pytest
import torch

from test_gpu_tc import CASES, FWD_ROWS, WG_ROWS, tc_pick_nt


def tc_pick_kc_tf32(cin):
    """csrc/conv_args.h tc_pick_kc_tf32: the largest multiple of 8 <= 32 dividing Cin"""
    return 0 if cin % 8 else next(kc for kc in (32, 24, 16, 8) if cin % kc == 0)


def tf32_rule(cin, cout, k, B):
    """the documented rule: the fp16 rule's kernel-size and batch limits with the TF32 channel table"""
    return (tc_pick_nt(cout) > 0 and tc_pick_kc_tf32(cin) > 0 and all(1 <= v <= 3 for v in k)
            and B * cin <= 4096 and B * cout <= 8192)


def _shapes():
    """every conv shape of test_gpu_tc's tables, both directions (data gradient: channels swap roles), plus the TF32
    channel table's edges"""
    out = set()
    for ci, co, k, shape, *_ in list(FWD_ROWS.values()) + list(CASES):
        out |= {(ci, co, k, shape[0]), (co, ci, k, shape[0])}
    for ci, co, k, shape in WG_ROWS.values():
        out |= {(ci, co, k, shape[0]), (co, ci, k, shape[0])}
    for ci in (8, 24, 40, 56, 72, 4, 12, 1):
        for co in (16, 8, 24, 144):
            for k in ((1, 1, 1), (1, 3, 3), (3, 3, 3), (5, 5, 5), (3, 1, 3)):
                for B in (1, 2, 64, 600):
                    out.add((ci, co, k, B))
    return sorted(out)


@pytest.fixture(scope="module")
def lib():
    from b200seg import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from b200seg.build import build
        build()
    return _lib.load()


@pytest.fixture
def precision():
    """sets torch.backends.cuda.matmul.fp32_precision for one test and restores exactly the saved value (other modules
    use the legacy getters, which raise while the new API's value is set)"""
    saved = torch.backends.cuda.matmul.fp32_precision

    def set_(v):
        torch.backends.cuda.matmul.fp32_precision = v
    yield set_
    torch.backends.cuda.matmul.fp32_precision = saved


def test_default_keeps_every_fp32_shape_direct(lib, precision):
    from b200seg import _lib, ops
    for value in (None, "ieee", "none"):
        if value is not None:
            precision(value)
        assert not ops.tf32_enabled()
        for ci, co, k, B in _shapes():
            assert ops.conv_algo(ci, co, k, torch.float32, B) == _lib.ALGO_DIRECT, (value, ci, co, k, B)
    # cuDNN's conv flag is not the switch
    assert torch.backends.cudnn.conv.fp32_precision == "tf32"
    assert ops.conv_algo(32, 32, (3, 3, 3), torch.float32, 1) == _lib.ALGO_DIRECT


@pytest.mark.parametrize("how", ["fp32_precision", "matmul_precision_high", "matmul_precision_medium", "allow_tf32"])
def test_tf32_follows_the_documented_rule(lib, precision, how):
    from b200seg import _lib, ops
    saved_legacy = torch.get_float32_matmul_precision()
    try:
        if how == "fp32_precision":
            precision("tf32")
        elif how == "allow_tf32":
            torch.backends.cuda.matmul.allow_tf32 = True
        else:
            torch.set_float32_matmul_precision(how.rsplit("_", 1)[1])
        assert ops.tf32_enabled()
        n_tc = 0
        for ci, co, k, B in _shapes():
            want = _lib.ALGO_TC_TF32 if tf32_rule(ci, co, k, B) else _lib.ALGO_DIRECT
            assert ops.conv_algo(ci, co, k, torch.float32, B) == want, (ci, co, k, B)
            assert lib.b200seg_conv3d_algo_tf32(ci, co, *k, B) == want
            # fp16 is untouched by the flag, and the fp16 query never answers TC for fp32
            assert ops.conv_algo(ci, co, k, torch.float16, B) == lib.b200seg_conv3d_algo(ci, co, *k, _lib.F16, B)
            assert lib.b200seg_conv3d_algo(ci, co, *k, _lib.F32, B) == _lib.ALGO_DIRECT
            n_tc += want == _lib.ALGO_TC_TF32
        assert n_tc > 100
    finally:
        if how != "fp32_precision":     # undo a legacy setter with the legacy API; the fixture then restores the value
            torch.set_float32_matmul_precision(saved_legacy)


def test_holder_repacks_when_the_flag_toggles(lib, precision, monkeypatch):
    """the chosen algorithms are part of a holder's signature: a toggle allocates a new image and packs it in the
    other layout; toggling back does the same again (never an image of one layout handed to the other kernel)"""
    from b200seg import _lib, ops
    packs = []
    monkeypatch.setattr(ops, "pack_weight", lambda w, dt, flip, out, off, co_total, layout: packs.append((flip, layout)))
    w1, w2 = torch.zeros(32, 16, 3, 3, 3), torch.zeros(16, 16, 3, 3, 3)     # fused conv1 + shortcut: co_total 48
    h = ops.PackedWeights()
    fwd, bwd = h.get([w1, w2], torch.float32)
    assert (fwd[1], bwd[1]) == (_lib.ALGO_DIRECT, _lib.ALGO_DIRECT)
    assert sorted(packs) == [(False, _lib.ALGO_DIRECT)] * 2 + [(True, _lib.ALGO_DIRECT)] * 2
    sig_exact = h._sig
    precision("tf32")
    packs.clear()
    fwd2, bwd2 = h.get([w1, w2], torch.float32)
    assert (fwd2[1], bwd2[1]) == (_lib.ALGO_TC_TF32, _lib.ALGO_TC_TF32)
    assert h._sig != sig_exact and fwd2[0] is not fwd[0] and bwd2[0] is not bwd[0]
    assert sorted(packs) == [(False, _lib.ALGO_TC_TF32)] * 2 + [(True, _lib.ALGO_TC_TF32)] * 2
    assert all(j[5] == _lib.ALGO_TC_TF32 for j in h._jobs)
    precision("ieee")
    packs.clear()
    fwd3, _ = h.get([w1, w2], torch.float32)
    assert fwd3[1] == _lib.ALGO_DIRECT and h._sig[:4] == sig_exact[:4]
    assert sorted(packs) == [(False, _lib.ALGO_DIRECT)] * 2 + [(True, _lib.ALGO_DIRECT)] * 2
    # fp16 holders keep their signature whatever the flag says
    h16 = ops.PackedWeights()
    h16.get([w1, w2], torch.float16)
    s16 = h16._sig
    precision("tf32")
    h16.get([w1, w2], torch.float16)
    assert h16._sig == s16


def test_pack_weight_rejects_mismatched_layouts(lib):
    """TC_TF32 images are fp32 only and TC images fp16 only; both need the tensor-core channel tables (checked before
    anything is launched, so no device is needed)"""
    from b200seg import _lib
    P = 16                       # a non-null placeholder: the calls below are rejected before any pointer is used
    assert lib.b200seg_pack_weight(P, 32, 16, 27, P, _lib.F16, 0, 0, 32, _lib.ALGO_TC_TF32, None) == -2
    assert lib.b200seg_pack_weight(P, 32, 16, 27, P, _lib.F32, 0, 0, 32, _lib.ALGO_TC, None) == -2
    assert lib.b200seg_pack_weight(P, 32, 12, 27, P, _lib.F32, 0, 0, 32, _lib.ALGO_TC_TF32, None) == -2
    assert lib.b200seg_pack_weight(P, 24, 16, 27, P, _lib.F32, 0, 0, 24, _lib.ALGO_TC_TF32, None) == -2
    assert lib.b200seg_pack_weight(P, 32, 16, 27, P, _lib.F32, 0, 0, 32, 4, None) == -1
