"""CPU: the ACDC MedFormer configuration on the host side.

  * get_model with the values of config/acdc/medformer_3d.yaml builds the reference's parameter set (the fixture's
    shapes), and the LiTS YAML's values (one head of 128..320 channels) still raise ValueError;
  * the ACDC forward / backward with every C-ABI op emulated (tests/emu_medformer.py, plus the wide B-MHA wrappers
    patched here) reproduces the reference fixture;
  * the B-MHA, map-generation and MHSA kernels compile without spills: every instantiation this configuration added
    reports 0 spill bytes, and the instantiations that were there before keep their register and spill counts."""
import importlib.util
import os
import re
import shutil
import subprocess
import types

import pytest
import torch

import b200seg
from oracle import losses as olosses
from oracle.synth import make_volume
from util import global_l2, load_golden, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "cbim-medical-image-segmentation_b200")


def _args(**over):
    """get_model's arguments with the values of config/acdc/medformer_3d.yaml (chan_num at MedFormer's default)"""
    a = dict(dimension="3d", model="medformer", in_chan=1, classes=4, base_chan=32, conv_block="BasicBlock",
             down_scale=[[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2]],
             kernel_size=[[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]], norm="in", act="relu",
             map_size=[2, 6, 6], conv_num=[2, 0, 0, 0, 0, 0, 2, 2], trans_num=[0, 2, 2, 2, 2, 2, 0, 0],
             num_heads=[1, 4, 4, 4, 4, 4, 1, 1], expansion=4, fusion_depth=2, fusion_dim=256, fusion_heads=4,
             attn_drop=0.0, proj_drop=0.0, proj_type="depthwise", aux_loss=True)
    a.update(over)
    return types.SimpleNamespace(**a)


def test_get_model_acdc_builds_the_reference_parameters():
    net = b200seg.get_model(_args())
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == load_golden("medformer_acdc")["shapes"]


def test_get_model_lits_still_raises():
    # config/lits/medformer_3d.yaml: map 4x4x4, one head per level (dim_head 128 / 256 / 320), fusion 320 / 10 heads
    lits = _args(map_size=[4, 4, 4], num_heads=[1, 1, 1, 1, 1, 1, 1, 1], fusion_dim=320, fusion_heads=10, classes=3)
    with pytest.raises(ValueError, match="dim_head"):
        b200seg.get_model(lits)


@pytest.mark.parametrize("over", [dict(map_size=[3, 6, 6]),                 # 108 map tokens
                                  dict(num_heads=[1, 4, 4, 4, 4, 2, 1, 1]),  # up2 at dim_head 64 is fine ...
                                  dict(num_heads=[1, 2, 4, 4, 4, 4, 1, 1]),  # ... down2 at 64 too; 128 is not:
                                  dict(num_heads=[1, 4, 2, 4, 4, 4, 1, 1]),
                                  dict(fusion_heads=8)])                     # 216 fused tokens at dim_head 32
def test_get_model_acdc_variants(over):
    ok = over.get("num_heads") in ([1, 4, 4, 4, 4, 2, 1, 1], [1, 2, 4, 4, 4, 4, 1, 1])
    if ok:
        b200seg.get_model(_args(**over))
    else:
        with pytest.raises(ValueError):
            b200seg.get_model(_args(**over))


def test_acdc_orchestration_matches_fixture(monkeypatch):
    """b200seg.MedFormer's ACDC wiring with every C-ABI op emulated reproduces the reference's logits and loss, and its
    gradients sit near the float64 oracle's (the GPU test holds the tight bar)."""
    import emu_medformer
    from b200seg import ops
    from oracle import medformer as omed
    from oracle.unet3d import make_state_dict
    emu_medformer.install(monkeypatch)
    # the wide B-MHA wrappers take the same emulation as the original pair
    monkeypatch.setattr(ops, "biattn_wide_fwd", ops.biattn_fwd)
    monkeypatch.setattr(ops, "biattn_wide_bwd", ops.biattn_bwd)
    g = load_golden("medformer_acdc")
    cfg = g["cfg"]
    kw = {k: cfg[k] for k in ("map_size", "conv_num", "trans_num", "num_heads", "fusion_depth", "fusion_dim",
                              "fusion_heads", "kernel_size", "scale", "aux_loss")}
    net = b200seg.MedFormer(1, cfg["classes"], 32, conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0,
                            proj_type="depthwise", norm="in", act="relu", **kw)
    sd = make_state_dict(g["shapes"], seed=cfg["state_seed"])
    for k in sd:
        if k.endswith("norm.weight"):
            sd[k] = 1.0 + 0.1 * sd[k] / sd[k].abs().max()
    net.load_state_dict(sd)
    img, lab = make_volume(*cfg["shape"], cfg["classes"], seed=cfg["data_seed"])
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    res = net(img)
    w = torch.tensor(cfg["ce_weight"])
    crit = b200seg.DiceCELoss(weight=w)
    loss = sum(cfg["aux_weight"][j] * crit(r, lab) for j, r in enumerate(res))
    loss.backward()
    for o, ref in zip(res, g["logits"]):
        assert o.shape == ref.shape and rel_err(o, ref.float()) < 2e-3          # fixture stored in fp16
    assert abs(loss.item() - g["loss"]) < 1e-4
    s64 = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    r64 = omed.medformer_forward(s64, img.double(), kw)
    olosses.total_loss(r64, lab, w.double(), cfg["aux_weight"]).backward()
    ours = {k: p.grad for k, p in net.named_parameters()}
    assert all(v is not None for v in ours.values())
    err = global_l2(ours, {k: v.grad for k, v in s64.items()})
    print("medformer_acdc emulated-orchestration grad L2 err vs fp64 oracle: %.2e" % err)
    assert err < 5e-2


# ============================================================================================ ptxas
# (registers, spill-store bytes, spill-load bytes) of every kernel of these files at the parent of the ACDC kernels,
# built with the library's flags; the keys are the mangled names without the anonymous-namespace prefix
PARENT = {
    "biattn.cu": {
        "biattn_bwd_kernelIfLi64EEEvNS_6BiArgsE": (255, 240, 240),
        "biattn_bwd_kernelIfLi32EEEvNS_6BiArgsE": (252, 0, 0),
        "biattn_bwd_kernelI6__halfLi64EEEvNS_6BiArgsE": (255, 244, 244),
        "biattn_bwd_kernelI6__halfLi32EEEvNS_6BiArgsE": (254, 0, 0),
        "biattn_bwd_merge_kernelIfEEvNS_6BiArgsEi": (32, 0, 0),
        "biattn_bwd_merge_kernelI6__halfEEvNS_6BiArgsEi": (32, 0, 0),
        "biattn_fwd_kernelIfLi64EEEvNS_6BiArgsE": (118, 0, 0),
        "biattn_fwd_kernelIfLi32EEEvNS_6BiArgsE": (88, 0, 0),
        "biattn_fwd_kernelI6__halfLi64EEEvNS_6BiArgsE": (116, 0, 0),
        "biattn_fwd_kernelI6__halfLi32EEEvNS_6BiArgsE": (86, 0, 0),
        "biattn_fwd_merge_kernelIfEEvNS_6BiArgsEi": (32, 0, 0),
        "biattn_fwd_merge_kernelI6__halfEEvNS_6BiArgsEi": (32, 0, 0),
    },
    "medformer_small.cu": {
        "mhsa_kernelIfEEvPKT_S3_PS1_S4_iif": (56, 0, 0),
        "mhsa_kernelI6__halfEEvPKT_S4_PS2_S5_iif": (56, 0, 0),
        "gelu_kernelIfEEvPKT_S3_PS1_l": (32, 0, 0),
        "gelu_kernelI6__halfEEvPKT_S4_PS2_l": (19, 0, 0),
        "layernorm_bwd_kernelIfEEvPKT_S3_PKfS5_PS1_PfS7_ii": (48, 0, 0),
        "layernorm_bwd_kernelI6__halfEEvPKT_S4_PKfS6_PS2_PfS8_ii": (43, 0, 0),
        "layernorm_fwd_kernelIfEEvPKT_PKfS5_PS1_Pfiif": (32, 0, 0),
        "layernorm_fwd_kernelI6__halfEEvPKT_PKfS6_PS2_Pfiif": (32, 0, 0),
        "scale_bwd_apply_kernelIfEEvPKT_PKfS5_PS1_lil": (32, 0, 0),
        "scale_bwd_apply_kernelI6__halfEEvPKT_PKfS6_PS2_lil": (32, 0, 0),
        "scale_bwd_reduce_kernelIfEEvPKT_S3_Pfli": (50, 0, 0),
        "scale_bwd_reduce_kernelI6__halfEEvPKT_S4_Pfli": (32, 0, 0),
        "scale_fwd_kernelIfEEvPKT_PKfPS1_lil": (32, 0, 0),
        "scale_fwd_kernelI6__halfEEvPKT_PKfPS2_lil": (32, 0, 0),
        "mapgen_bwd_kernelIfLi64EEEvNS_6MgArgsE": (167, 0, 0),
        "mapgen_bwd_kernelIfLi32EEEvNS_6MgArgsE": (110, 0, 0),
        "mapgen_bwd_kernelI6__halfLi64EEEvNS_6MgArgsE": (167, 0, 0),
        "mapgen_bwd_kernelI6__halfLi32EEEvNS_6MgArgsE": (103, 0, 0),
        "mapgen_fwd_kernelIfLi64EEEvNS_6MgArgsE": (96, 0, 0),
        "mapgen_fwd_kernelIfLi32EEEvNS_6MgArgsE": (56, 0, 0),
        "mapgen_fwd_kernelI6__halfLi64EEEvNS_6MgArgsE": (106, 0, 0),
        "mapgen_fwd_kernelI6__halfLi32EEEvNS_6MgArgsE": (56, 0, 0),
        "mapgen_merge_kernelIfEEvNS_6MgArgsEi": (32, 0, 0),
        "mapgen_merge_kernelI6__halfEEvNS_6MgArgsEi": (32, 0, 0),
        "s2d_kernelIfLi1EEEvPKT_PS1_iiiiiiiii": (34, 0, 0),
        "s2d_kernelI6__halfLi1EEEvPKT_PS2_iiiiiiiii": (34, 0, 0),
        "s2d_kernelIfLi8EEEvPKT_PS1_iiiiiiiii": (32, 0, 0),
        "s2d_kernelI6__halfLi8EEEvPKT_PS2_iiiiiiiii": (32, 0, 0),
        "scale_bwd_sum_kernelEPKfPfii": (32, 0, 0),
        "se_gate_bwd_kernelENS_6SeArgsE": (40, 0, 0),
        "se_gate_fwd_kernelENS_6SeArgsE": (40, 0, 0),
    },
}
# name prefixes of the instantiations added for ACDC: the wide B-MHA, the dim_head 64 MHSA, the 80-code map generation
NEW = {"biattn.cu": ("biattn_wide_",),
       "medformer_small.cu": ("mhsa64_kernel", "mapgen_fwd_kernelIfLi80", "mapgen_fwd_kernelI6__halfLi80",
                              "mapgen_bwd_kernelIfLi80", "mapgen_bwd_kernelI6__halfLi80")}


def _ptxas(src, tmp_path):
    nvcc = os.environ.get("NVCC", "nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("nvcc not found")
    spec = importlib.util.spec_from_file_location("_b200seg_build_acdc", os.path.join(PKG, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    cmd = [nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(b.CSRC, src), "-o", str(tmp_path / (src + ".o"))]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    out, cur, spill = {}, None, None
    for line in r.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            k = re.search(r"_cu_[0-9a-f]{8}\d+(\w+)$", m.group(1))
            cur = k.group(1) if k else m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            spill = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur and spill is not None:
            out[cur] = (int(m.group(1)), *spill)
            cur, spill = None, None
    return out


@pytest.mark.parametrize("src", ["biattn.cu", "medformer_small.cu"])
def test_ptxas_new_kernels_do_not_spill_and_old_ones_are_unchanged(src, tmp_path):
    rep = _ptxas(src, tmp_path)
    parent = PARENT[src]
    new = {k: v for k, v in rep.items() if any(k.startswith(p) for p in NEW[src])}
    print("%s new instantiations: %s" % (src, new))
    assert new, "no new instantiation in the ptxas report of %s" % src
    assert all(v[1] == 0 and v[2] == 0 for v in new.values()), new
    old = {k: v for k, v in rep.items() if k not in new}
    assert old == parent, {k: (old.get(k), parent.get(k)) for k in set(old) | set(parent) if old.get(k) != parent.get(k)}
