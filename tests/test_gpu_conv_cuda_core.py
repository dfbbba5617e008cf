"""The CUDA-core convolutions (csrc/conv_direct.cu) and the HBM-bound special cases (csrc/small_conv.cu) against
PyTorch float64, on every kernel instantiation and at the shapes the benchmark sends them.

Every AMP step runs the stems and classifier heads here, and an fp32 step runs every convolution on conv_direct.cu.
Each table runs in fp32 and fp16 (ALGO_DIRECT forward, ALGO_AUTO weight gradient unless a row says otherwise):
  STEM_ROWS  stem_fwd_kernel<T, KD, KH, KW, NG>: the Cin = 1 forward with fused InstanceNorm sums.  1x3x3 / 3x3x3 /
             1x1x1 x Cout 32 / 48 / 64 (all 18 instantiations), V not a multiple of 256, B = 2, D = 1 under 3x3x3, the
             output a slice (y_ld = Cout + 16, y_coff = 8) with a sentinel around it and NaN in it.  One row has a CT-like
             input (3 + 0.05 randn: the outputs' |mean| is 60x their std), which a 1e-5 error in the raw sums of squares
             would turn into a large variance error.
  PW_ROWS    pointwise_small_kernel<T, CIN>: the 1x1x1 head forward and its data gradient.  CIN 4 / 8 / 16 / 32 / 64 x
             Cout 4 / 32 / 64, with and without bias, dense or sliced x and y.
  CIN1_ROWS  wgrad_cin1_kernel<T, KD, KH, KW, TWO>: the stem weight gradient.  Each kernel with Cout 16 / 32 (one lane
             half) and 40 / 48 / 64 (a second half, partly empty below 64); W = 300 (two 256-column chunks, the halo
             across the seam), H = 13 (a partial 8-row group), B = 2, D = 1 under 3x3x3.
  HEAD_ROWS  wgrad_head_kernel<T, MAXCO, CPT>: the 1x1x1 head weight and bias gradient, <4, 8> and <16, 2>.  Cout 1 / 2
             / 3 / 4 (the vector dy load, and a sliced dy without it) / 5 / 14 / 16; Cin 8 / 24 / 40 / 48 / 56 / 128 (24,
             40, 48 and 56 leave lanes of the 256 idle); raw, or InstanceNorm + ReLU / LeakyReLU input; bias or not.
             In fp16 the tensor cores take Cout = 16 with Cin = 48 / 128, so those rows are left out (route_wgrad).
  DF_ROWS    conv_fwd_direct_kernel<T, CIV>: CIV 8 (Cin 32) and CIV 1 (Cin 3 / 14) in the five modes of test_gpu_tc.py
             (bias; IN + ReLU + residual + sums; IN + LeakyReLU + sums; data gradient with the ReLU / LeakyReLU mask),
             Cout 3 / 14 / 17 / 33 against the 16-channel tile, 1x1x1 / 1x3x3 / 3x3x3, V = 351 (not a multiple of 128).
             5x5x5 with CIV 8 takes 64 KB of shared memory (the opt-in branch), 7x7x7 172 KB; 9x9x9 is refused.
  DW_ROWS    conv_wgrad_direct_kernel<T> (ALGO_DIRECT): Cin x Cout over 1 / 3 / 14 / 33 / 40 against the 32-wide tiles,
             raw or IN + ReLU / LeakyReLU input, bias, three voxel chunks per block column, and 5x5x5.  B * coT * ciT >
             65535 is refused.
  PACK_ROWS  pack_weight_kernel<T>: the DIRECT layout, plain and transpose_flip, inside a co_off / co_total window, bit
             for bit against a torch permute / flip.
  FULL_FWD, FULL_WG: every shape one AMP step of resunet_acdc_128, resunet_kits_160, swin_unetr_amos_128 and
             medformer_bcv_96 sends to these kernels (test_bench_shapes_are_full_size_rows records them), at full size:
             the persistent weight-gradient kernels then have more jobs than blocks.
  MISALIGNED: the stem and the pointwise head on tensors whose storage starts one element past a 16-byte boundary.
             Their vector stores and loads cannot take such a base, so these calls go to conv_fwd_direct_kernel.
  test_tables_reach_every_instantiation (CPU) mirrors the host-side routing (route_fwd / route_wgrad) and checks that
  the tables reach all 18 + 10 + 12 + 4 special-kernel instantiations and all 4 + 2 CUDA-core ones;
  test_rows_launch_the_mirrored_kernel checks the kernel names the profiler sees.

Reference: float64 on the device (never TF32) on the kernel's own inputs and dtype-rounded weights, rounded to the
storage dtype where the kernel rounds: the normalised, activated loader operand, the conv output before a residual add,
and the masked data gradient.  Each output is judged against its own max (util.rel_err's metric): y, dw, dbias.  The
fused InstanceNorm sums are judged through what they are used for: the mean in units of the channel's std, and the
variance against its own max; data-gradient sums (sum g, sum g*h) against their own max.  Elements whose data-gradient
mask input is within MASK_MARGIN of 0 are left out.  The bars (BARS) are the largest errors measured on an H100 80GB
HBM3 at 700 W with at most 3x headroom; DESIGN.md section 4 lists them.
"""
import zlib

import pytest
import torch
import torch.nn.functional as F

from util import SENTINEL, assert_untouched, launched_kernels_each, run_fresh, wide

gpu = pytest.mark.gpu

EPS = 1e-4
MASK_MARGIN = 1e-3
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2          # B200SEG_ACT_*
ALGO_AUTO, ALGO_DIRECT, ALGO_TC = 0, 1, 2        # B200SEG_ALGO_*
NUM_SMS = 132                                    # B200SEG_NUM_SMS
DTS = ("fp32", "fp16")
TNAME = {"fp32": "float", "fp16": "__half"}
K111, K133, K333, K555, K777, K999 = (1, 1, 1), (1, 3, 3), (3, 3, 3), (5, 5, 5), (7, 7, 7), (9, 9, 9)

# bars: (table, dtype) -> {output: bar}; the largest error measured on an H100 80GB HBM3 (700 W) is in the comments
BARS = {
    ("stem", "fp32"): dict(y=6e-7, mean=6e-8, var=1.2e-7),             # 2.2e-7, 2.3e-8, 4.2e-8
    ("stem", "fp16"): dict(y=1e-3, mean=6e-9, var=1e-7),               # 3.9e-4, 2.1e-9, 3.8e-8
    ("stem_ct", "fp32"): dict(y=9e-8, mean=5e-6, var=1.5e-4),          # 3.1e-8, 1.7e-6, 5.6e-5
    ("stem_ct", "fp16"): dict(y=1e-3, mean=5e-6, var=1.5e-4),          # 3.3e-4, 0 (exact), 5.9e-5
    ("pw", "fp32"): dict(y=1e-6),                                       # 4.0e-7
    ("pw", "fp16"): dict(y=1e-3),                                       # 4.2e-4
    ("cin1", "fp32"): dict(dw=1.5e-6),                                  # 5.0e-7
    ("cin1", "fp16"): dict(dw=1.2e-6),                                  # 4.1e-7
    ("head", "fp32"): dict(dw=3e-6, db=2.5e-6),                         # 1.2e-6, 9.2e-7
    ("head", "fp16"): dict(dw=1.2e-4, db=2e-5),                         # 4.9e-5, 7.8e-6
    ("df", "fp32"): dict(y=3.5e-6, mean=1.2e-7, var=2.5e-7, gsum=6e-7),  # 1.3e-6, 4.4e-8, 9.8e-8, 2.4e-7
    ("df", "fp16"): dict(y=1e-3, mean=2.4e-8, var=2e-7, gsum=6e-7),      # 4.8e-4, 8.0e-9, 7.4e-8, 2.6e-7
    ("df_big", "fp32"): dict(y=1.2e-5, mean=1.2e-7, var=2.5e-7, gsum=6e-7),   # 5x5x5 / 7x7x7: 4.1e-6
    ("df_big", "fp16"): dict(y=1e-3, mean=2.4e-8, var=2e-7, gsum=6e-7),       # 4.3e-4
    ("dw", "fp32"): dict(dw=3e-6, db=3e-5),                             # 1.2e-6, 1.2e-5 (Cout = 1: one cancelling sum)
    ("dw", "fp16"): dict(dw=9e-5, db=5e-6),                             # 3.1e-5, 1.9e-6
    ("full", "fp16"): dict(y=1e-3, mean=5e-11, var=3e-8, dw=2e-6, db=1.4e-6),  # 4.2e-4, 1.7e-11, 1.1e-8, 7.8e-7, 4.8e-7
}


# ----------------------------------------------------------------------------- host-side routing, mirrored
def pick_ntc(cin):
    """csrc/wgrad_tc.cu pick_ntc"""
    if cin % 16:
        return 0
    if cin % 128 == 0:
        return 64
    if cin <= 128:
        return cin
    return next((v for v in (128, 96, 64, 48, 32, 16) if cin % v == 0), 0)


def _esz(dt):
    return 2 if dt == "fp16" else 4


def route_fwd(dt, Cin, Cout, k, plain, bias, stats, x_ld, x_coff, y_ld, y_coff, x_addr=0, y_addr=0):
    """The kernel an ALGO_DIRECT b200seg_conv3d_fwd launches (csrc/small_conv.cu conv3d_fwd_small, then
    csrc/conv_direct.cu conv3d_fwd_direct), or None when it refuses the shape.  plain: no input normalisation or
    activation, no residual, not in data-gradient mode; x_addr / y_addr: the base addresses (only their alignment
    matters)."""
    T, vec4 = TNAME[dt], 4 * _esz(dt)
    if (plain and not bias and Cin == 1 and Cout in (32, 48, 64) and k in (K133, K333, K111) and y_ld % 8 == 0
            and y_coff % 8 == 0 and y_addr % 16 == 0):
        return "stem_fwd_kernel<%s, %d, %d, %d, %d>" % (T, *k, Cout // 16)
    if (plain and not stats and k == K111 and Cin in (4, 8, 16, 32, 64) and Cout % 4 == 0 and Cout <= 64
            and x_ld % 4 == 0 and x_coff % 4 == 0 and y_ld % 4 == 0 and y_coff % 4 == 0
            and x_addr % vec4 == 0 and y_addr % vec4 == 0):
        return "pointwise_small_kernel<%s, %d>" % (T, Cin)
    civ8 = Cin % 8 == 0 and x_ld % 8 == 0 and x_coff % 8 == 0 and x_addr % 16 == 0
    civ = 8 if civ8 else 1
    if 4 * (k[0] * k[1] * k[2] * 16 * civ + 2 * Cin + 4 * 16 * 2) > 200 * 1024:
        return None
    return "conv_fwd_direct_kernel<%s, %d>" % (T, civ)


def wgrad_tc_takes(dt, B, Cin, Cout, k, x_ld, x_coff, dy_ld, dy_coff, x_addr, dy_addr):
    """csrc/wgrad_tc.cu conv3d_wgrad_tc_supported without its bias condition (every shape here fits the stage ring)"""
    return (dt == "fp16" and max(k) <= 3 and x_ld % 8 == 0 and x_coff % 8 == 0 and dy_ld % 8 == 0 and dy_coff % 8 == 0
            and x_addr % 16 == 0 and dy_addr % 16 == 0 and pick_ntc(Cin) > 0 and Cout % 8 == 0
            and B * pick_ntc(Cin) <= 2048)


def route_wgrad(dt, B, Cin, Cout, k, norm, act, bias, x_ld, x_coff, dy_ld, dy_coff, algo=ALGO_AUTO, x_addr=0,
                dy_addr=0):
    """The kernel b200seg_conv3d_wgrad launches (csrc/api.cu: tensor cores, tensor cores after a separate bias pass when
    Cout % 8 == 0, then small_wgrad_kind in csrc/small_conv.cu, then csrc/conv_direct.cu), or None when it refuses."""
    T = TNAME[dt]
    if algo == ALGO_AUTO:
        if wgrad_tc_takes(dt, B, Cin, Cout, k, x_ld, x_coff, dy_ld, dy_coff, x_addr, dy_addr) and (not bias or Cout % 8 == 0):
            return "wgrad_tc_kernel"
        if Cin == 1 and Cout <= 64 and k in (K133, K333, K111) and not norm and not act and not bias:
            return "wgrad_cin1_kernel<%s, %d, %d, %d, %s>" % (T, *k, "true" if Cout > 32 else "false")
        if (k == K111 and Cout <= 16 and Cin <= 128 and Cin % 8 == 0 and x_ld % 8 == 0 and x_coff % 8 == 0
                and x_addr % 16 == 0):
            return "wgrad_head_kernel<%s, %s>" % (T, "4, 8" if Cout <= 4 else "16, 2")
    if B * -(-Cout // 32) * -(-Cin // 32) > 65535:
        return None
    return "conv_wgrad_direct_kernel<%s>" % T


# ----------------------------------------------------------------------------- tables
STEM_GEOM = (2, 3, 11, 13)                         # V = 429 per batch
STEM_ROWS = {}                                     # name: (Cout, k, (B, D, H, W), CT-like input)
for _k, _kn in ((K133, "k133"), (K333, "k333"), (K111, "k111")):
    for _co in (32, 48, 64):
        STEM_ROWS["%s_co%d" % (_kn, _co)] = (_co, _k, STEM_GEOM, False)
STEM_ROWS["k333_co32_d1"] = (32, K333, (2, 1, 11, 13), False)
STEM_ROWS["k333_co64_d1"] = (64, K333, (2, 1, 11, 13), False)
STEM_ROWS["ct_k111_co48"] = (48, K111, STEM_GEOM, True)

PW_GEOM = (2, 3, 7, 13)
PW_ROWS = {}                                       # name: (Cin, Cout, bias, sliced)
for _ci in (4, 8, 16, 32, 64):
    for _co in (4, 32, 64):
        for _b in (False, True):
            for _s in (False, True):
                PW_ROWS["ci%d_co%d_%s_%s" % (_ci, _co, "bias" if _b else "nobias", "sliced" if _s else "dense")] = (_ci, _co, _b, _s)

CIN1_ROWS = {}                                     # name: (Cout, k, (B, D, H, W))
for _k, _kn in ((K133, "k133"), (K333, "k333"), (K111, "k111")):
    for _co in (16, 32, 40, 48, 64):
        CIN1_ROWS["%s_co%d" % (_kn, _co)] = (_co, _k, (2, 3, 13, 300))
CIN1_ROWS["k333_co16_d1"] = (16, K333, (2, 1, 13, 300))
CIN1_ROWS["k333_co48_d1"] = (48, K333, (2, 1, 13, 300))

HEAD_GEOM = (2, 3, 17, 23)
HEAD_COUTS = {"co1": (1, None), "co2": (2, None), "co3": (3, None), "co4v": (4, None), "co4s": (4, (6, 2)),
              "co5": (5, None), "co14": (14, None), "co16": (16, None)}       # (Cout, (dy_ld, dy_coff) or dense)
HEAD_INPUTS = {"raw_bias": (ACT_NONE, True), "raw": (ACT_NONE, False), "relu_bias": (ACT_RELU, True),
               "lrelu": (ACT_LRELU, False)}                                    # (IN + act or raw, bias)
HEAD_ROWS = {}                                     # name: (Cin, Cout, dy slice, act, bias)
for _cn, (_co, _sl) in HEAD_COUTS.items():
    for _ci in (8, 24, 40, 48, 56, 128):
        for _in, (_a, _b) in HEAD_INPUTS.items():
            HEAD_ROWS["%s_ci%d_%s" % (_cn, _ci, _in)] = (_ci, _co, _sl, _a, _b)

DF_GEOM = (2, 3, 9, 13)                            # V = 351 per batch
DF_MODES = ("bias", "relu_res", "lrelu", "dgrad_relu", "dgrad_lrelu")
DF_ROWS = {}                                       # name: (Cin, Cout, k, (B, D, H, W), mode)
for _ci in (3, 14, 32):
    for _co in (3, 14, 17, 33):
        for _k, _kn in ((K111, "k111"), (K133, "k133"), (K333, "k333")):
            for _m in DF_MODES:
                DF_ROWS["ci%d_co%d_%s-%s" % (_ci, _co, _kn, _m)] = (_ci, _co, _k, DF_GEOM, _m)
for _k, _kn, _sh in ((K555, "k555", (1, 5, 9, 11)), (K777, "k777", (1, 7, 9, 11))):
    for _m in ("relu_res", "dgrad_lrelu"):
        DF_ROWS["ci32_co17_%s-%s" % (_kn, _m)] = (32, 17, _k, _sh, _m)

DW_GEOM = (2, 5, 19, 31)                           # V = 2945: three 1024-voxel chunks per (tap, tile) column
DW_INPUTS = {"raw_bias": (ACT_NONE, True), "relu": (ACT_RELU, False), "lrelu_bias": (ACT_LRELU, True)}
DW_ROWS = {}                                       # name: (Cin, Cout, k, (B, D, H, W), act, bias)
for _ci in (1, 3, 14, 33, 40):
    for _co in (1, 3, 14, 33, 40):
        for _in, (_a, _b) in DW_INPUTS.items():
            DW_ROWS["ci%d_co%d_%s" % (_ci, _co, _in)] = (_ci, _co, K333, DW_GEOM, _a, _b)
DW_ROWS["ci14_co33_k555_lrelu_bias"] = (14, 33, K555, (1, 6, 12, 14), ACT_LRELU, True)

PACK_ROWS = {                                      # name: (Cout, Cin, k, co_off, co_total)
    "co3_ci14_k333": (3, 14, K333, 0, 3), "co3_ci14_k333_window": (3, 14, K333, 5, 12),
    "co33_ci1_k133": (33, 1, K133, 0, 33), "co33_ci1_k133_window": (33, 1, K133, 2, 40),
    "co16_ci32_k111_window": (16, 32, K111, 16, 48), "co40_ci3_k555_window": (40, 3, K555, 1, 41),
}

# the pointwise head and the stem with their base one element past a 16-byte boundary: (table row, x / y misaligned)
MISALIGNED = {"stem_k133_co32": ("k133_co32", True, True), "stem_k333_co48": ("k333_co48", True, True),
              "stem_k111_co64_y": ("k111_co64", False, True), "pw_ci32_co4_bias": ("ci32_co4_bias_dense", True, True),
              "pw_ci4_co32": ("ci4_co32_nobias_dense", True, False), "pw_ci64_co64_y": ("ci64_co64_bias_dense", False, True)}

# the benchmark's own calls (test_bench_shapes_are_full_size_rows): fp16, dense operands
FULL_FWD = {       # name: (Cin, Cout, k, (B, D, H, W), mode)   mode: stats (stem) / bias (head) / plain (head dgrad)
    "acdc_stem": (1, 32, K133, (1, 128, 128, 128), "stats"),
    "acdc_head": (32, 4, K111, (1, 128, 128, 128), "bias"),
    "acdc_head_dgrad": (4, 32, K111, (1, 128, 128, 128), "plain"),
    "kits_stem": (1, 32, K333, (2, 160, 160, 80), "stats"),
    "kits_head": (32, 3, K111, (2, 160, 160, 80), "bias"),
    "kits_head_dgrad": (3, 32, K111, (2, 160, 160, 80), "plain"),
    "swin_enc1": (1, 48, K333, (1, 128, 128, 128), "stats"),
    "swin_enc1_proj": (1, 48, K111, (1, 128, 128, 128), "stats"),
    "swin_patch_embed": (8, 48, K111, (1, 64, 64, 64), "bias"),
    "med_stem": (1, 32, K133, (1, 96, 96, 96), "stats"),
    "med_head": (32, 14, K111, (1, 96, 96, 96), "bias"),
    "med_head_dgrad": (14, 32, K111, (1, 96, 96, 96), "plain"),
}
FULL_WG = {        # name: (Cin, Cout, k, (B, D, H, W), bias)
    "acdc_stem": (1, 32, K133, (1, 128, 128, 128), False),
    "acdc_head": (32, 4, K111, (1, 128, 128, 128), True),
    "kits_stem": (1, 32, K333, (2, 160, 160, 80), False),
    "kits_head": (32, 3, K111, (2, 160, 160, 80), True),
    "swin_enc1": (1, 48, K333, (1, 128, 128, 128), False),
    "swin_enc1_proj": (1, 48, K111, (1, 128, 128, 128), False),
    "swin_patch_embed": (8, 48, K111, (1, 64, 64, 64), True),
    "med_stem": (1, 32, K133, (1, 96, 96, 96), False),
    "med_head": (32, 14, K111, (1, 96, 96, 96), True),
}
BENCH = ("resunet_acdc_128", "resunet_kits_160", "swin_unetr_amos_128", "medformer_bcv_96")


def _fwd_route_row(table, row, dt):
    """route_fwd of a forward table row as the tests below launch it"""
    if table == "stem":
        Cout, k, _, _ = STEM_ROWS[row]
        return route_fwd(dt, 1, Cout, k, True, False, True, 1, 0, Cout + 16, 8)
    if table == "pw":
        Cin, Cout, bias, sl = PW_ROWS[row]
        return route_fwd(dt, Cin, Cout, K111, True, bias, False, *_pw_layout(Cin, Cout, sl))
    if table == "df":
        Cin, Cout, k, _, mode = DF_ROWS[row]
        return route_fwd(dt, Cin, Cout, k, False, mode == "bias", mode != "bias", Cin, 0, Cout, 0)
    if table == "mis":
        base, xm, ym = MISALIGNED[row]
        e = _esz(dt)
        if row.startswith("stem"):
            Cout, k, _, _ = STEM_ROWS[base]
            return route_fwd(dt, 1, Cout, k, True, False, True, 1, 0, Cout, 0, e * xm, e * ym)
        Cin, Cout, bias, _ = PW_ROWS[base]
        return route_fwd(dt, Cin, Cout, K111, True, bias, False, Cin, 0, Cout, 0, e * xm, e * ym)
    Cin, Cout, k, _, mode = FULL_FWD[row]
    return route_fwd(dt, Cin, Cout, k, True, mode == "bias", mode == "stats", Cin, 0, Cout, 0)


def _wg_route_row(table, row, dt):
    if table == "cin1":
        Cout, k, (B, *_) = CIN1_ROWS[row]
        return route_wgrad(dt, B, 1, Cout, k, False, ACT_NONE, False, 1, 0, Cout, 0)
    if table == "head":
        Cin, Cout, sl, act, bias = HEAD_ROWS[row]
        dy_ld, dy_coff = sl or (Cout, 0)
        return route_wgrad(dt, HEAD_GEOM[0], Cin, Cout, K111, act != ACT_NONE, act, bias, Cin, 0, dy_ld, dy_coff)
    if table == "dw":
        Cin, Cout, k, (B, *_), act, bias = DW_ROWS[row]
        return route_wgrad(dt, B, Cin, Cout, k, act != ACT_NONE, act, bias, Cin, 0, Cout, 0, algo=ALGO_DIRECT)
    Cin, Cout, k, (B, *_), bias = FULL_WG[row]
    return route_wgrad(dt, B, Cin, Cout, k, False, ACT_NONE, bias, Cin, 0, Cout, 0)


def _pw_layout(Cin, Cout, sliced):
    """(x_ld, x_coff, y_ld, y_coff) of a pointwise row"""
    return (Cin + 8, 4, Cout + 8, 4) if sliced else (Cin, 0, Cout, 0)


HEAD_REACHABLE = [(r, dt) for r in HEAD_ROWS for dt in DTS if _wg_route_row("head", r, dt).startswith("wgrad_head")]


# ----------------------------------------------------------------------------- CPU: the tables cover the library
def test_tables_reach_every_instantiation():
    fwd = {}
    for table, rows in (("stem", STEM_ROWS), ("pw", PW_ROWS), ("df", DF_ROWS), ("mis", MISALIGNED)):
        for r in rows:
            for dt in DTS:
                fwd.setdefault(table, set()).add(_fwd_route_row(table, r, dt))
    want_stem = {"stem_fwd_kernel<%s, %d, %d, %d, %d>" % (TNAME[dt], *k, ng)
                 for dt in DTS for k in (K133, K333, K111) for ng in (2, 3, 4)}
    want_pw = {"pointwise_small_kernel<%s, %d>" % (TNAME[dt], c) for dt in DTS for c in (4, 8, 16, 32, 64)}
    want_df = {"conv_fwd_direct_kernel<%s, %d>" % (TNAME[dt], c) for dt in DTS for c in (1, 8)}
    assert len(want_stem) == 18 and len(want_pw) == 10
    assert fwd["stem"] == want_stem and fwd["pw"] == want_pw, (fwd["stem"] ^ want_stem, fwd["pw"] ^ want_pw)
    assert fwd["df"] == want_df
    # the misaligned rows: the stem and the pointwise head would take them without their base-address conditions
    assert fwd["mis"] <= want_df and {d for d in fwd["mis"] if d.endswith("8>")}, fwd["mis"]
    for r, (base, xm, ym) in MISALIGNED.items():
        table = "stem" if r.startswith("stem") else "pw"
        assert _fwd_route_row(table, base, "fp16").startswith("stem_fwd" if table == "stem" else "pointwise_small")
    # the refusal of more than 200 KB of shared memory: 9x9x9 with CIV 8
    assert route_fwd("fp16", 32, 17, K999, False, False, True, 32, 0, 17, 0) is None
    assert route_fwd("fp16", 32, 17, K777, False, False, True, 32, 0, 17, 0) is not None

    cin1 = {_wg_route_row("cin1", r, dt) for r in CIN1_ROWS for dt in DTS}
    want_cin1 = {"wgrad_cin1_kernel<%s, %d, %d, %d, %s>" % (TNAME[dt], *k, two)
                 for dt in DTS for k in (K133, K333, K111) for two in ("true", "false")}
    assert len(want_cin1) == 12 and cin1 == want_cin1, cin1 ^ want_cin1
    head = {_wg_route_row("head", r, dt) for r, dt in HEAD_REACHABLE}
    want_head = {"wgrad_head_kernel<%s, %s>" % (TNAME[dt], b) for dt in DTS for b in ("4, 8", "16, 2")}
    assert head == want_head
    assert {_wg_route_row("head", r, dt) for r in HEAD_ROWS for dt in DTS} - head == {"wgrad_tc_kernel"}
    assert {_wg_route_row("dw", r, dt) for r in DW_ROWS for dt in DTS} == {"conv_wgrad_direct_kernel<%s>" % TNAME[dt] for dt in DTS}
    assert route_wgrad("fp32", 65536, 1, 1, K111, False, ACT_NONE, False, 1, 0, 1, 0, algo=ALGO_DIRECT) is None
    assert route_wgrad("fp32", 65535, 1, 1, K111, False, ACT_NONE, False, 1, 0, 1, 0, algo=ALGO_DIRECT) is not None
    # the cin1 rows need two column chunks and a partial row group; the head rows idle lanes of the 256 threads
    assert all(s[3] > 256 and s[2] % 8 for _, _, s in CIN1_ROWS.values())
    assert {256 % (ci // (8 if co <= 4 else 2)) != 0 for ci, co, *_ in HEAD_ROWS.values()} == {False, True}
    # the full-size rows take the special kernels or the CUDA cores, never the tensor cores
    for r in FULL_FWD:
        assert _fwd_route_row("full", r, "fp16") is not None
    for r in FULL_WG:
        assert _wg_route_row("full", r, "fp16") != "wgrad_tc_kernel", r


@pytest.fixture(scope="module")
def host_lib():
    import os
    from b200seg import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from b200seg.build import build
        build()
    return _lib.load()


def test_head_workspace_matches_mirror(host_lib):
    """the library sizes the weight-gradient workspace for the kernel the mirror names: a head / stem slice per
    persistent block, or nothing for the CUDA-core kernel"""
    for r, dt in HEAD_REACHABLE:
        Cin, Cout, sl, act, bias = HEAD_ROWS[r]
        dy_ld, dy_coff = sl or (Cout, 0)
        got = host_lib.b200seg_conv3d_wgrad_workspace(Cin, 0, int(act != ACT_NONE), dy_ld, dy_coff, int(bias), *HEAD_GEOM,
                                                      Cin, Cout, 1, 1, 1, 1 if dt == "fp16" else 0, ALGO_AUTO)
        assert got == NUM_SMS * 2 * (Cout * Cin + Cout) * 4, r
    for r in CIN1_ROWS:
        Cout, k, shape = CIN1_ROWS[r]
        got = host_lib.b200seg_conv3d_wgrad_workspace(1, 0, 0, Cout, 0, 0, *shape, 1, Cout, *k, 1, ALGO_AUTO)
        assert got == NUM_SMS * 2 * Cout * k[0] * k[1] * k[2] * 4, r


# ----------------------------------------------------------------------------- inputs and references
@pytest.fixture(autouse=True)
def no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def seed_of(name):
    return zlib.crc32(name.encode()) & 0x7fffffff


def _dtype(dt):
    return torch.float16 if dt == "fp16" else torch.float32


def randt(shape, dt, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale + offset).to(_dtype(dt)).cuda()


def randf(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def misaligned_like(t):
    """t's values in storage that starts one element past a 16-byte boundary"""
    buf = torch.empty(t.numel() + 8, dtype=t.dtype, device=t.device)
    out = buf[1:1 + t.numel()].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16
    return out


def nan_slice(lead, ld, coff, C, dtype):
    """an output buffer: a sentinel outside channels coff .. coff+C, NaN inside"""
    y = torch.full((*lead, ld), SENTINEL, dtype=dtype, device="cuda")
    y[..., coff:coff + C] = float("nan")
    return y


def nc(t):
    """[B, D, H, W, C] -> float64 [B, C, D, H, W] on the device"""
    return t.double().permute(0, 4, 1, 2, 3)


def rerr(a, ref):
    """max-norm relative error ||a - ref||_inf / ||ref||_inf on the device (NaN anywhere fails every bar)"""
    a, ref = a.double(), ref.double()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def stats64(t):
    d = t.double().flatten(1, 3)
    return torch.stack([d.sum(1), (d * d).sum(1)], -1)


def xhat64(t, st):
    n = t[0, ..., 0].numel()
    m = st[..., 0] / n
    r = 1.0 / torch.sqrt((st[..., 1] / n - m * m).clamp_min(0) + EPS)
    return (nc(t) - m[:, :, None, None, None]) * r[:, :, None, None, None]


def act64(h, act):
    return h if act == ACT_NONE else (h.clamp_min(0) if act == ACT_RELU else torch.where(h > 0, h, 0.01 * h))


def dact64(h, act):
    one = torch.ones_like(h)
    return one if act == ACT_NONE else torch.where(h > 0, one, (0.0 if act == ACT_RELU else 0.01) * one)


def rnd(t, dt):
    return t.to(_dtype(dt)).double()


def loader64(x, xst, act, dt):
    """what the kernels stage: x itself, or dt(act(IN(x)))"""
    if xst is None and act == ACT_NONE:
        return nc(x)
    return rnd(act64(xhat64(x, xst) if xst is not None else nc(x), act), dt)


def conv64(a, w, k, dt, bias=None):
    return F.conv3d(a, rnd(w, dt), None if bias is None else bias.double(), padding=[i // 2 for i in k])


def wgrad64(a, dy, Cout, k):
    """dW[co, ci, tap] = sum_v dy[v, co] * a[v + tap, ci] as one fp64 product per tap of dy with a shifted, zero-padded
    view of a (a: [B, Cin, D, H, W] float64; dy: [B, D, H, W, Cout])"""
    B, Cin, D, H, W = a.shape
    p = [i // 2 for i in k]
    ap = F.pad(a, (p[2], p[2], p[1], p[1], p[0], p[0]))
    g = dy.double().reshape(-1, Cout)
    dw = torch.empty(Cout, Cin, *k, dtype=torch.float64, device=a.device)
    for zd in range(k[0]):
        for zh in range(k[1]):
            for zw in range(k[2]):
                s = ap[:, :, zd:zd + D, zh:zh + H, zw:zw + W].permute(0, 2, 3, 4, 1).reshape(-1, Cin)
                dw[:, :, zd, zh, zw] = g.t() @ s
    return dw


def stats_errs(st, y, h=None):
    """the fused InstanceNorm sums st [B, C, 2] against the stored y: (mean error in units of the channel std, variance
    error against the largest variance), or in data-gradient mode (sum g, sum g*h) against their own max"""
    st = st.double()
    if h is not None:
        g = nc(y)
        ref = torch.stack([g.sum((2, 3, 4)), (g * h).sum((2, 3, 4))], -1)
        return dict(gsum=max(rerr(st[..., 0], ref[..., 0]), rerr(st[..., 1], ref[..., 1])))
    n = y[0, ..., 0].numel()
    y64 = y.double().flatten(1, 3)
    m_ref = y64.mean(1)
    v_ref = ((y64 - m_ref[:, None, :]) ** 2).mean(1)
    m = st[..., 0] / n
    v = st[..., 1] / n - m * m
    return dict(mean=((m - m_ref).abs() / v_ref.sqrt().clamp_min(1e-30)).max().item(), var=rerr(v, v_ref))


def judge(record, table, dt, **errs):
    bars = BARS[(table, dt)]
    for name, e in errs.items():
        record(name + "_err", e)
    bad = {n: e for n, e in errs.items() if not e < bars[n]}
    assert not bad, (bad, {n: bars[n] for n in bad})


def _p(t):
    return None if t is None else t.data_ptr()


def fwd_raw(x, x_ld, x_coff, xst, act, wp, y, y_ld, y_coff, yst, Cin, Cout, k, shape, bias=None, res=None, r_ld=0,
            r_coff=0, dg=None):
    """b200seg_conv3d_fwd (ALGO_DIRECT) on caller-provided buffers"""
    from b200seg import _lib, ops
    gx, g_ld, g_coff, gst, gact = dg or (None, 0, 0, None, ACT_NONE)
    _lib.call("b200seg_conv3d_fwd", x.data_ptr(), x_ld, x_coff, _p(xst), EPS, act, wp.data_ptr(), _p(bias), _p(res),
              r_ld, r_coff, y.data_ptr(), y_ld, y_coff, _p(yst), _p(gx), g_ld, g_coff, _p(gst), EPS, gact, *shape,
              Cin, Cout, *k, ops._dt(x), ALGO_DIRECT, ops._stream())


def wgrad_raw(x, x_ld, x_coff, xst, act, dy, dy_ld, dy_coff, dw, db, Cin, Cout, k, shape, algo=ALGO_AUTO):
    """b200seg_conv3d_wgrad into caller-provided dw / dbias (added to, not overwritten)"""
    from b200seg import _lib, ops
    ws_bytes = _lib.load().b200seg_conv3d_wgrad_workspace(x_ld, x_coff, int(xst is not None or act != ACT_NONE), dy_ld,
                                                          dy_coff, int(db is not None), *shape, Cin, Cout, *k,
                                                          ops._dt(x), algo)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device="cuda")
    _lib.call("b200seg_conv3d_wgrad", x.data_ptr(), x_ld, x_coff, _p(xst), EPS, act, dy.data_ptr(), dy_ld, dy_coff,
              dw.data_ptr(), _p(db), *shape, Cin, Cout, *k, ops._dt(x), algo, ws.data_ptr(), ws_bytes, ops._stream())


def pack(w, dt):
    from b200seg import ops
    return ops.pack_weight(w, _dtype(dt))


# ----------------------------------------------------------------------------- launches (also run under the profiler)
def launch_stem(row, dt, misaligned=(False, False)):
    Cout, k, shape, ct = STEM_ROWS[row]
    s = seed_of(row + dt)
    taps = k[0] * k[1] * k[2]
    x = randt((*shape, 1), dt, s, scale=0.05 if ct else 1.0, offset=3.0 if ct else 0.0)
    w = randf(Cout, 1, *k, seed=s + 1) / taps ** 0.5
    if any(misaligned):
        y_ld, y_coff = Cout, 0
        y = nan_slice(shape, y_ld, 0, Cout, _dtype(dt))
        xk = misaligned_like(x) if misaligned[0] else x
        y = misaligned_like(y) if misaligned[1] else y
    else:
        y_ld, y_coff, xk = Cout + 16, 8, x
        y = nan_slice(shape, y_ld, y_coff, Cout, _dtype(dt))
    st = torch.zeros(shape[0], Cout, 2, dtype=torch.float64, device="cuda")
    fwd_raw(xk, 1, 0, None, ACT_NONE, pack(w, dt), y, y_ld, y_coff, st, 1, Cout, k, shape)
    return dict(x=x, w=w, y=y, y_coff=y_coff, st=st, Cout=Cout, k=k)


def launch_pw(row, dt, misaligned=(False, False)):
    Cin, Cout, bias, sliced = PW_ROWS[row]
    s = seed_of(row + dt)
    x = randt((*PW_GEOM, Cin), dt, s)
    w = randf(Cout, Cin, 1, 1, 1, seed=s + 1) / Cin ** 0.5
    b = randf(Cout, seed=s + 2) if bias else None
    x_ld, x_coff, y_ld, y_coff = _pw_layout(Cin, Cout, sliced)
    xk = wide(x, x_ld, x_coff)
    y = nan_slice(PW_GEOM, y_ld, y_coff, Cout, _dtype(dt))
    if misaligned[0]:
        xk = misaligned_like(xk)
    if misaligned[1]:
        y = misaligned_like(y)
    fwd_raw(xk, x_ld, x_coff, None, ACT_NONE, pack(w, dt), y, y_ld, y_coff, None, Cin, Cout, K111, PW_GEOM, bias=b)
    return dict(x=x, w=w, b=b, y=y, y_coff=y_coff, Cout=Cout)


def launch_mis(row, dt):
    base, xm, ym = MISALIGNED[row]
    return (launch_stem if row.startswith("stem") else launch_pw)(base, dt, (xm, ym))


def _df_inputs(row, dt):
    Cin, Cout, k, shape, mode = DF_ROWS[row]
    s = seed_of(row + dt)
    taps = k[0] * k[1] * k[2]
    inp = dict(x=randt((*shape, Cin), dt, s), w=randf(Cout, Cin, *k, seed=s + 1) / (Cin * taps) ** 0.5, xst=None,
               act=ACT_NONE, bias=None, res=None, dg=None, stats=mode != "bias")
    if mode == "bias":
        inp["bias"] = randf(Cout, seed=s + 2, scale=0.5)
    elif mode in ("relu_res", "lrelu"):
        inp.update(xst=stats64(inp["x"]), act=ACT_RELU if mode == "relu_res" else ACT_LRELU)
        if mode == "relu_res":
            inp["res"] = randt((*shape, Cout), dt, s + 3)
    else:
        gx = randt((*shape, Cout), dt, s + 4)
        inp["dg"] = (gx, Cout, 0, stats64(gx), ACT_RELU if mode == "dgrad_relu" else ACT_LRELU)
    return inp


def launch_df(row, dt):
    Cin, Cout, k, shape, mode = DF_ROWS[row]
    inp = _df_inputs(row, dt)
    y = nan_slice(shape, Cout, 0, Cout, _dtype(dt))
    st = torch.zeros(shape[0], Cout, 2, dtype=torch.float64, device="cuda") if inp["stats"] else None
    fwd_raw(inp["x"], Cin, 0, inp["xst"], inp["act"], pack(inp["w"], dt), y, Cout, 0, st, Cin, Cout, k, shape,
            bias=inp["bias"], res=inp["res"], r_ld=Cout, dg=inp["dg"])
    inp.update(y=y, st=st)
    return inp


def _wg_case(x, xst, act, dy, dy_ld, dy_coff, Cin, Cout, k, shape, bias, seed, algo):
    """dw (and dbias) twice from zero and once into non-zero buffers"""
    dw0 = randf(Cout, Cin, *k, seed=seed + 7, scale=0.1)
    db0 = randf(Cout, seed=seed + 8, scale=10.0) if bias else None
    runs = []
    for _ in range(2):
        runs.append((torch.zeros_like(dw0), torch.zeros_like(db0) if bias else None))
        wgrad_raw(x, Cin, 0, xst, act, dy, dy_ld, dy_coff, *runs[-1], Cin, Cout, k, shape, algo)
    acc = (dw0.clone(), db0.clone() if bias else None)
    wgrad_raw(x, Cin, 0, xst, act, dy, dy_ld, dy_coff, *acc, Cin, Cout, k, shape, algo)
    return dict(runs=runs, acc=acc, dw0=dw0, db0=db0)


def launch_cin1(row, dt):
    Cout, k, shape = CIN1_ROWS[row]
    s = seed_of(row + dt)
    x = randt((*shape, 1), dt, s)
    dy = randt((*shape, Cout), dt, s + 1)
    out = _wg_case(x, None, ACT_NONE, dy, Cout, 0, 1, Cout, k, shape, False, s, ALGO_AUTO)
    out.update(x=x, dy=dy)
    return out


def launch_head(row, dt):
    Cin, Cout, sl, act, bias = HEAD_ROWS[row]
    s = seed_of(row + dt)
    x = randt((*HEAD_GEOM, Cin), dt, s, scale=2.0, offset=0.5)
    dy = randt((*HEAD_GEOM, Cout), dt, s + 1)
    xst = stats64(x) if act != ACT_NONE else None
    dy_ld, dy_coff = sl or (Cout, 0)
    out = _wg_case(x, xst, act, wide(dy, dy_ld, dy_coff), dy_ld, dy_coff, Cin, Cout, K111, HEAD_GEOM, bias, s, ALGO_AUTO)
    out.update(x=x, xst=xst, dy=dy)
    return out


def launch_dw(row, dt):
    Cin, Cout, k, shape, act, bias = DW_ROWS[row]
    s = seed_of(row + dt)
    x = randt((*shape, Cin), dt, s, scale=2.0, offset=0.5)
    dy = randt((*shape, Cout), dt, s + 1)
    xst = stats64(x) if act != ACT_NONE else None
    out = _wg_case(x, xst, act, dy, Cout, 0, Cin, Cout, k, shape, bias, s, ALGO_DIRECT)
    out.update(x=x, xst=xst, dy=dy)
    return out


def launch(table, row, dt):
    """one table row's launches (the profiler test runs this in a fresh process)"""
    return {"stem": launch_stem, "pw": launch_pw, "mis": launch_mis, "df": launch_df, "cin1": launch_cin1,
            "head": launch_head, "dw": launch_dw}[table](row, dt)


# ----------------------------------------------------------------------------- forward tables
def _check_stem(out, dt, table, record):
    y = out["y"]
    assert_untouched(y, out["y_coff"], out["Cout"])
    ys = y[..., out["y_coff"]:out["y_coff"] + out["Cout"]]
    ref = conv64(nc(out["x"]), out["w"], out["k"], dt)
    judge(record, table, dt, y=rerr(nc(ys), ref), **stats_errs(out["st"], ys))
    return ys


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(STEM_ROWS))
def test_stem_fwd(row, dt, record_property):
    out = launch_stem(row, dt)
    torch.cuda.synchronize()
    ct = STEM_ROWS[row][3]
    ys = _check_stem(out, dt, "stem_ct" if ct else "stem", record_property)
    if ct:
        y64 = ys.double().flatten(1, 3)
        assert (y64.mean(1).abs() >= 50 * y64.std(1)).all()


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(PW_ROWS))
def test_pointwise_fwd(row, dt, record_property):
    out = launch_pw(row, dt)
    torch.cuda.synchronize()
    Cout, y_coff = out["Cout"], out["y_coff"]
    assert_untouched(out["y"], y_coff, Cout)
    ref = conv64(nc(out["x"]), out["w"], K111, dt, out["b"])
    judge(record_property, "pw", dt, y=rerr(nc(out["y"][..., y_coff:y_coff + Cout]), ref))


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(MISALIGNED))
def test_misaligned_base(row, dt, record_property):
    """a base address the vector accesses cannot take: the call goes to the CUDA-core kernel and gives the fp64 answer"""
    out = launch_mis(row, dt)
    torch.cuda.synchronize()
    if row.startswith("stem"):
        _check_stem(out, dt, "stem", record_property)
    else:
        ref = conv64(nc(out["x"]), out["w"], K111, dt, out["b"])
        judge(record_property, "pw", dt, y=rerr(nc(out["y"]), ref))


def _df_ref(inp, dt, k, act=None, g_act=None):
    act = inp["act"] if act is None else act
    y = conv64(loader64(inp["x"], inp["xst"], act, dt), inp["w"], k, dt, inp["bias"])
    if inp["res"] is not None:
        y = rnd(y, dt) + nc(inp["res"])
    if inp["dg"] is None:
        return y, torch.ones_like(y, dtype=torch.bool), None
    gx, _, _, gst, ga = inp["dg"]
    h = xhat64(gx, gst)
    return y * dact64(h, ga if g_act is None else g_act), h.abs() >= MASK_MARGIN, h


def _masked(y, ref, keep):
    return rerr(torch.where(keep, y, 0.0), torch.where(keep, ref, 0.0))


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(DF_ROWS))
def test_direct_fwd(row, dt, record_property):
    Cin, Cout, k, shape, mode = DF_ROWS[row]
    out = launch_df(row, dt)
    torch.cuda.synchronize()
    ref, keep, h = _df_ref(out, dt, k)
    y = nc(out["y"])
    errs = dict(y=_masked(y, ref, keep))
    if out["st"] is not None:
        errs.update(stats_errs(out["st"], out["y"], h))
    table = "df_big" if max(k) > 3 else "df"
    judge(record_property, table, dt, **errs)
    if mode in ("lrelu", "dgrad_lrelu"):          # the row can see the LeakyReLU slope
        twin, _, _ = _df_ref(out, dt, k, act=ACT_RELU if mode == "lrelu" else None, g_act=ACT_RELU)
        assert _masked(twin, ref, keep) > 3 * BARS[(table, dt)]["y"]


@gpu
@pytest.mark.parametrize("dt", DTS)
def test_direct_fwd_refuses_over_200kb(dt):
    """9x9x9 with CIV 8 needs 373 KB of shared memory: EUNSUPPORTED before anything is launched"""
    from b200seg import _lib
    shape, Cin, Cout = (1, 3, 5, 7), 32, 17
    x = randt((*shape, Cin), dt, 1)
    wp = pack(randf(Cout, Cin, *K999, seed=2), dt)
    y = nan_slice(shape, Cout + 8, 8, 0, _dtype(dt))
    with pytest.raises(_lib.B200SegError, match="not supported"):
        fwd_raw(x, Cin, 0, None, ACT_NONE, wp, y, Cout + 8, 8, None, Cin, Cout, K999, shape)
    torch.cuda.synchronize()
    assert_untouched(y, 0, 0)


# ----------------------------------------------------------------------------- weight-gradient tables
def _check_wg(out, ref_dw, ref_db, table, dt, record, exact):
    (dw, db), (dw2, db2) = out["runs"]
    dwa, dba = out["acc"]
    if exact:            # per-block partials summed in block order, then added to what dw / dbias hold
        assert torch.equal(dw, dw2) and torch.equal(dwa, out["dw0"] + dw)
        if ref_db is not None:
            assert torch.equal(db, db2) and torch.equal(dba, out["db0"] + db)
    errs = dict(dw=max(rerr(dw, ref_dw), rerr(dwa.double() - out["dw0"].double(), ref_dw)))
    if ref_db is not None:
        errs["db"] = max(rerr(db, ref_db), rerr(dba.double() - out["db0"].double(), ref_db))
    judge(record, table, dt, **errs)


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(CIN1_ROWS))
def test_stem_wgrad(row, dt, record_property):
    Cout, k, _ = CIN1_ROWS[row]
    out = launch_cin1(row, dt)
    torch.cuda.synchronize()
    _check_wg(out, wgrad64(nc(out["x"]), out["dy"], Cout, k), None, "cin1", dt, record_property, exact=True)


@gpu
@pytest.mark.parametrize("row,dt", HEAD_REACHABLE)
def test_head_wgrad(row, dt, record_property):
    Cin, Cout, _, act, bias = HEAD_ROWS[row]
    out = launch_head(row, dt)
    torch.cuda.synchronize()
    a = loader64(out["x"], out["xst"], act, dt)
    ref = wgrad64(a, out["dy"], Cout, K111)
    _check_wg(out, ref, nc(out["dy"]).sum((0, 2, 3, 4)) if bias else None, "head", dt, record_property, exact=True)
    if act == ACT_LRELU:
        assert rerr(wgrad64(loader64(out["x"], out["xst"], ACT_RELU, dt), out["dy"], Cout, K111), ref) > \
            3 * BARS[("head", dt)]["dw"]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(DW_ROWS))
def test_direct_wgrad(row, dt, record_property):
    """float atomics: compared with fp64, never bit for bit"""
    Cin, Cout, k, _, act, bias = DW_ROWS[row]
    out = launch_dw(row, dt)
    torch.cuda.synchronize()
    ref = wgrad64(loader64(out["x"], out["xst"], act, dt), out["dy"], Cout, k)
    _check_wg(out, ref, nc(out["dy"]).sum((0, 2, 3, 4)) if bias else None, "dw", dt, record_property, exact=False)


@gpu
def test_direct_wgrad_refuses_zblocks():
    """B * coT * ciT = 65536 z-blocks: EUNSUPPORTED, dw untouched"""
    from b200seg import _lib
    shape = (65536, 1, 1, 1)
    x = randt((*shape, 1), "fp32", 3)
    dy = randt((*shape, 1), "fp32", 4)
    dw = torch.full((1, 1, 1, 1, 1), 7.0, device="cuda")
    with pytest.raises(_lib.B200SegError, match="not supported"):
        wgrad_raw(x, 1, 0, None, ACT_NONE, dy, 1, 0, dw, None, 1, 1, K111, shape, ALGO_DIRECT)
    torch.cuda.synchronize()
    assert dw.item() == 7.0


@gpu
@pytest.mark.parametrize("tf", [False, True])
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", list(PACK_ROWS))
def test_pack_weight_direct(row, dt, tf):
    """the DIRECT image [tap][co_total][Cin] (forward) or [flipped tap][Cin][co_total] (data gradient), bit for bit"""
    from b200seg import ops
    Cout, Cin, k, co_off, co_total = PACK_ROWS[row]
    taps = k[0] * k[1] * k[2]
    w = randf(Cout, Cin, *k, seed=seed_of(row))
    dtype = _dtype(dt)
    shape = (taps, Cin, co_total) if tf else (taps, co_total, Cin)
    out = torch.full(shape, SENTINEL, dtype=dtype, device="cuda")
    ops.pack_weight(w, dtype, transpose_flip=tf, out=out, co_off=co_off, co_total=co_total)
    torch.cuda.synchronize()
    want = torch.full(shape, SENTINEL, dtype=dtype, device="cuda")
    if tf:
        want[:, :, co_off:co_off + Cout] = w.flip(2, 3, 4).permute(2, 3, 4, 1, 0).reshape(taps, Cin, Cout).to(dtype)
    else:
        want[:, co_off:co_off + Cout, :] = w.permute(2, 3, 4, 0, 1).reshape(taps, Cout, Cin).to(dtype)
    assert torch.equal(out, want)


# ----------------------------------------------------------------------------- which kernel each row launches
_FAMILIES = ("stem_fwd_kernel", "pointwise_small_kernel", "conv_fwd_direct_kernel", "wgrad_cin1_kernel",
             "wgrad_head_kernel", "conv_wgrad_direct_kernel", "wgrad_tc_kernel")


def _norm_name(n):
    return n.replace(" ", "").replace("(int)", "").replace("(bool)", "")


def _profiled_rows():
    """one row per instantiation of each table (the first that reaches it), and every misaligned row"""
    rows, seen = [], set()
    for table, names in (("stem", STEM_ROWS), ("pw", PW_ROWS), ("df", DF_ROWS), ("cin1", CIN1_ROWS),
                         ("head", HEAD_ROWS), ("dw", DW_ROWS), ("mis", MISALIGNED)):
        for r in names:
            for dt in DTS:
                kern = (_wg_route_row(table, r, dt) if table in ("cin1", "head", "dw") else _fwd_route_row(table, r, dt))
                if table == "mis" or (kern not in seen and kern != "wgrad_tc_kernel"):
                    seen.add(kern)
                    rows.append((table, r, dt, kern))
    return rows


def _ours(names):
    return {_norm_name(n) for n in names if any(f in n for f in _FAMILIES)}


@gpu
def test_rows_launch_the_mirrored_kernel():
    rows = _profiled_rows()
    calls = [("launch", (t, r, dt)) for t, r, dt, _ in rows]
    names = []
    for i in range(0, len(calls), 16):      # a few sessions per process: a long series of sessions can lose launches
        names += launched_kernels_each("test_gpu_conv_cuda_core", calls[i:i + 16])
    # now and then a session comes back without its kernel records: such a row is profiled once more
    lost = [i for i, got in enumerate(names) if not _ours(got)]
    if lost:
        for i, got in zip(lost, launched_kernels_each("test_gpu_conv_cuda_core", [calls[i] for i in lost])):
            names[i] = got
    for (table, r, dt, kern), got in zip(rows, names):
        ours = _ours(got)
        assert ours and all(_norm_name(kern) in n for n in ours), (table, r, dt, kern, sorted(ours))


# ----------------------------------------------------------------------------- the benchmark's shapes
def _mode_of(bias, yst, gx, xst, act, res):
    if gx or xst or act or res:
        return "other"
    return "bias" if bias else ("stats" if yst else "plain")


def record_bench_calls(workload):
    """every b200seg_conv3d_fwd / b200seg_conv3d_wgrad call of one AMP TrainStep of a bench.py workload that routes to
    small_conv.cu or conv_direct.cu, as [kind, kernel, Cin, Cout, k, (B, D, H, W), mode or bias]"""
    import bench
    import b200seg
    from b200seg import ops
    from b200seg.train import TrainStep
    from oracle.synth import make_volume
    wl = bench.WORKLOADS[workload]
    scale, kernel, classes, weight, (B, D, H, W) = wl
    dev = torch.device("cuda")

    def make_net():
        if bench.is_swin(wl):
            n = b200seg.SwinUNETR((D, H, W), 1, classes, feature_size=wl[1])
            n.load_state_dict(bench.oracle_state(wl), strict=False)
            return n.to(dev)
        if bench.is_medformer(wl):
            n = b200seg.MedFormer(1, classes, bench.BASE, conv_block="BasicBlock", expansion=4, attn_drop=0, proj_drop=0,
                                  proj_type="depthwise", norm="in", act="relu", **wl[0])
        else:
            n = b200seg.UNet(1, bench.BASE, scale=scale, kernel_size=kernel, num_classes=classes, block="BasicBlock",
                             norm="in")
        n.load_state_dict(bench.oracle_state(wl))
        return n.to(dev)
    net, ema = make_net(), make_net()
    for p in ema.parameters():
        p.requires_grad_(False)
    ts = TrainStep(net, ema, ce_weight=torch.tensor(weight), amp=True,
                   aux_weight=bench.AUX_WEIGHT if bench.is_medformer(wl) else None)
    img, lab = make_volume(B, D, H, W, classes, seed=2023)
    seen = set()
    real = ops.call

    def call(name, *a):
        if name == "b200seg_conv3d_fwd" and a[31] == ALGO_DIRECT:
            dt = "fp16" if a[30] == 1 else "fp32"
            Cin, Cout, k = a[25], a[26], tuple(a[27:30])
            plain = not (a[3] or a[5] or a[8] or a[15])
            kern = route_fwd(dt, Cin, Cout, k, plain, bool(a[7]), bool(a[14]), a[1], a[2], a[12], a[13], a[0], a[11])
            if dt == "fp16" and (a[1], a[2], a[12], a[13]) == (Cin, 0, Cout, 0):
                seen.add(("fwd", kern, Cin, Cout, k, tuple(a[21:25]), _mode_of(a[7], a[14], a[15], a[3], a[5], a[8])))
            else:
                seen.add(("fwd_other", kern, Cin, Cout, k, tuple(a[21:25]), dt))
        elif name == "b200seg_conv3d_wgrad":
            dt = "fp16" if a[20] == 1 else "fp32"
            Cin, Cout, k, shape = a[15], a[16], tuple(a[17:20]), tuple(a[11:15])
            kern = route_wgrad(dt, shape[0], Cin, Cout, k, bool(a[3]), a[5], bool(a[10]), a[1], a[2], a[7], a[8],
                               a[21], a[0], a[6])
            if kern != "wgrad_tc_kernel":
                ok = dt == "fp16" and not (a[3] or a[5]) and (a[1], a[2], a[7], a[8]) == (Cin, 0, Cout, 0)
                seen.add(("wgrad" if ok else "wgrad_other", kern, Cin, Cout, k, shape, bool(a[10])))
        return real(name, *a)
    ops.call = call
    try:
        ts(img.to(dev), lab.to(dev))
        torch.cuda.synchronize()
    finally:
        ops.call = real
    return sorted((list(t) for t in seen), key=str)


def _full_keys():
    keys = set()
    for r, (Cin, Cout, k, shape, mode) in FULL_FWD.items():
        keys.add(("fwd", _fwd_route_row("full", r, "fp16"), Cin, Cout, k, shape, mode))
    for r, (Cin, Cout, k, shape, bias) in FULL_WG.items():
        keys.add(("wgrad", _wg_route_row("full", r, "fp16"), Cin, Cout, k, shape, bias))
    return keys


@gpu
@pytest.mark.parametrize("workload", BENCH)
def test_bench_shapes_are_full_size_rows(workload):
    """one AMP step of the benchmarked workload, recorded in a process of its own: every call it sends to
    small_conv.cu or conv_direct.cu is a row of FULL_FWD / FULL_WG"""
    got = {tuple(tuple(v) if isinstance(v, list) else v for v in t) for t in run_fresh("test_gpu_conv_cuda_core",
                                                                                       "record_bench_calls", workload)}
    print("%s: %s" % (workload, sorted(got, key=str)))
    assert got, "the step sent nothing to these kernels"
    assert got <= _full_keys(), sorted(got - _full_keys(), key=str)


def _full_ref_fwd(row):
    Cin, Cout, k, shape, mode = FULL_FWD[row]
    s = seed_of(row)
    x = randt((*shape, Cin), "fp16", s)
    w = randf(Cout, Cin, *k, seed=s + 1) / (Cin * k[0] * k[1] * k[2]) ** 0.5
    b = randf(Cout, seed=s + 2) if mode == "bias" else None
    st = torch.zeros(shape[0], Cout, 2, dtype=torch.float64, device="cuda") if mode == "stats" else None
    y = nan_slice(shape, Cout, 0, Cout, torch.float16)
    fwd_raw(x, Cin, 0, None, ACT_NONE, pack(w, "fp16"), y, Cout, 0, st, Cin, Cout, k, shape, bias=b)
    torch.cuda.synchronize()
    errs = dict(y=rerr(nc(y), conv64(nc(x), w, k, "fp16", b)))
    if st is not None:
        errs.update(stats_errs(st, y))
    return errs


@gpu
@pytest.mark.parametrize("row", list(FULL_FWD))
def test_full_size_fwd(row, record_property):
    judge(record_property, "full", "fp16", **_full_ref_fwd(row))
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("row", list(FULL_WG))
def test_full_size_wgrad(row, record_property):
    """the persistent stem and head kernels with more jobs than blocks, and the swin patch embedding on the CUDA cores"""
    Cin, Cout, k, shape, bias = FULL_WG[row]
    s = seed_of(row)
    x = randt((*shape, Cin), "fp16", s)
    dy = randt((*shape, Cout), "fp16", s + 1)
    dw = torch.zeros(Cout, Cin, *k, device="cuda")
    db = torch.zeros(Cout, device="cuda") if bias else None
    wgrad_raw(x, Cin, 0, None, ACT_NONE, dy, Cout, 0, dw, db, Cin, Cout, k, shape)
    torch.cuda.synchronize()
    errs = dict(dw=rerr(dw, wgrad64(nc(x), dy, Cout, k)))
    if bias:
        errs["db"] = rerr(db, dy.double().sum((0, 1, 2, 3)))
    judge(record_property, "full", "fp16", **errs)
    torch.cuda.empty_cache()
