"""The wgmma implicit-GEMM convolutions (ALGO_TC) against PyTorch float64, on every kernel instantiation and across the
mechanisms they have.

The forward / data-gradient kernel is one instantiation conv_tc_kernel<NT, KSTEPS> per N tile NT = tc_pick_nt(Cout)
and K chunk KSTEPS = tc_pick_kc(Cin) / 16 (csrc/conv_tc.cu).  The weight-gradient kernel dispatches once per CTA to
consumer_role<NTC, NTAPS>: Cin tile NTC = pick_ntc(Cin), NTAPS = the in-plane taps of the job's group (fill_params in
csrc/wgrad_tc.cu).  Each instantiation has its own register allocation, wgmma specialisation and unrolled epilogue, so
each one is run here:
  * FWD_ROWS: all 32 (NT, KSTEPS) on a base shape (Cin = 16 KSTEPS, Cout = NT, 3x3x3, (B, D, H, W) = (2, 3, 20, 12):
    ragged 16 x 8 tiles, depth taps outside the volume, a batch boundary inside a CTA's tile walk) in five modes:
      bias         raw x, bias, no statistics          raw tensor-TMA loader, bias epilogue
      relu_res     IN + ReLU, residual, statistics     normalising loader, residual epilogue, InstanceNorm sums
      lrelu        IN + LeakyReLU, statistics          norm_act8<false>
      dgrad_relu   data-gradient mode, ReLU mask       dgrad mask, both IN-backward sums
      dgrad_lrelu  data-gradient mode, LeakyReLU       act_grad_s with slope 0.01
    plus several N tiles per NT (bias / statistics / s_gnorm offsets of later N tiles), several K chunks per KSTEPS with
    Cin > 64 (cp.async loader), the asymmetric kernels 1x1x3 / 1x3x1 / 3x1x1, LeakyReLU without statistics (mean 0,
    rstd 1) and D = 1 on the raw TMA path.  The weights are resident for small layers and streamed for large ones.
  * WG_ROWS: every reachable (NTC, NTAPS), one Cin tile and several, with Cout = 16 / 48 (second consumer warpgroup
    idle), 72 (8 real rows in it), 128, 136 / 200 (a second M tile of 8 / 72 rows), each with ACT_NONE and with ReLU /
    LeakyReLU on InstanceNorm statistics.  WG_EDGE_ROWS: split-K S == 1 (>= 132 jobs; one voxel tile) and S > 1,
    D = 1 with kd = 3 (jobs that own no valid tile), accumulation into a non-zero dw, bit-identical repeats.
  * test_tables_reach_every_instantiation (CPU) mirrors the host-side tiling choices and checks that these tables reach
    every instantiation the library can launch; test_every_conv_tc_instantiation_launches checks the forward names the
    profiler sees.

Reference: float64 on the same fp16 inputs, rounded to fp16 exactly where the kernel rounds (the normalised, activated
loader output; the conv output before a residual add), computed on the device in float64 (never TF32).  Bars, max-norm
(util.rel_err):
  * forward / data gradient FWD_BAR = 1e-3 against the unrounded fp64 result: one half-ulp of fp16 (2^-11 relative) per
    stored rounding, two with a residual (largest observed 6.2e-4).  A pre-activation within rounding of 0 may legitimately take either branch of
    the data-gradient mask, so elements with |h| < MASK_MARGIN are left out of that max.
  * InstanceNorm sums of the output against the sums of the stored y: 1e-5.
  * weight gradient: dw is accumulated and stored in fp32.  On raw inputs only the fp32 sums separate it from fp64
    (largest observed error 1.7e-6, bar WG_BAR_RAW = 1e-5).  Behind the normalising loader a staged value whose fp32
    normalisation lands on the other side of an fp16 rounding boundary than the fp64 one differs by one ulp; one such
    element under a large dy moves a dw entry by up to ~1e-4 of the largest (largest observed 1.04e-4, bar
    WG_BAR = 3e-4).  Observed on an H100 80GB HBM3 at a 700 W power limit.
  * every LeakyReLU row first checks that its reference differs from the ReLU one by more than 3x the bar, i.e. that the
    row can see the slope.
"""
import re
import zlib

import pytest
import torch
import torch.nn.functional as F

from util import rel_err

gpu = pytest.mark.gpu

EPS = 1e-4
FWD_BAR = 1e-3
STATS_BAR = 1e-5
WG_BAR_RAW, WG_BAR = 1e-5, 3e-4
MASK_MARGIN = 1e-3
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2        # B200SEG_ACT_*

# ----------------------------------------------------------------------------- host-side tiling choices, mirrored
NUM_SMS = 132                                  # B200SEG_NUM_SMS, csrc/common.cuh


def tc_pick_nt(cout):
    """csrc/conv_args.h tc_pick_nt: whole Cout up to 128, else the largest even split into multiples of 16 <= 128"""
    if cout % 16:
        return 0
    if cout <= 128:
        return cout
    for t in range((cout + 127) // 128, 33):
        if cout % t == 0 and (cout // t) % 16 == 0 and cout // t <= 128:
            return cout // t
    return 0


def tc_pick_kc(cin):
    """csrc/conv_args.h tc_pick_kc: the largest multiple of 16 <= 64 dividing Cin"""
    return 0 if cin % 16 else next(kc for kc in (64, 48, 32, 16) if cin % kc == 0)


def pick_ntc(cin):
    """csrc/wgrad_tc.cu pick_ntc"""
    if cin % 16:
        return 0
    if cin % 128 == 0:
        return 64
    if cin <= 128:
        return cin
    return next((v for v in (128, 96, 64, 48, 32, 16) if cin % v == 0), 0)


def wg_plan(cin, cout, k, shape):
    """csrc/wgrad_tc.cu fill_params: ({(NTC, NTAPS)} of the consumers the jobs run, split-K factor S)"""
    kd, kh, kw = k
    B, D, H, W = shape
    ntc = pick_ntc(cin)
    taps_hw = kh * kw
    g = min(192 // ntc, taps_hw)                                   # kMaxCols / NTC
    ngroups = -(-taps_hw // g)
    gbase, grem = divmod(taps_hw, ngroups)
    consumers = {(ntc, gbase)} | ({(ntc, gbase + 1)} if grem else set())
    jobs = -(-cout // 128) * (cin // ntc) * kd * ngroups
    nvt = B * D * -(-H // 16) * -(-W // 8)
    return consumers, min(max(1, NUM_SMS // jobs), nvt)


def fwd_inst(cin, cout):
    return tc_pick_nt(cout), tc_pick_kc(cin) // 16


# ----------------------------------------------------------------------------- tables
K3 = (3, 3, 3)
BASE = (2, 3, 20, 12)
NTS = (16, 32, 48, 64, 80, 96, 112, 128)
FWD_MODES = ("bias", "relu_res", "lrelu", "dgrad_relu", "dgrad_lrelu")
MULTI_MODES = ("bias", "relu_res", "dgrad_lrelu")

FWD_ROWS = {}      # name: (Cin, Cout, k, (B, D, H, W), mode)
for _nt in NTS:
    for _ks in (1, 2, 3, 4):
        for _m in FWD_MODES:
            FWD_ROWS["nt%d_ks%d-%s" % (_nt, _ks, _m)] = (16 * _ks, _nt, K3, BASE, _m)
# NTILES > 1: one Cout per NT (tc_pick_nt(Cout) = NT)
for _nt, _co in zip(NTS, (176, 352, 144, 704, 160, 192, 224, 256)):
    for _m in MULTI_MODES:
        FWD_ROWS["ntiles_co%d-%s" % (_co, _m)] = (48, _co, K3, BASE, _m)
# NKC > 1, Cin > 64 (cp.async loader when normalised): one Cin per KSTEPS
for _ci in (80, 160, 144, 128):
    for _m in MULTI_MODES:
        FWD_ROWS["nkc_ci%d-%s" % (_ci, _m)] = (_ci, 64, K3, BASE, _m)
for _k in ((1, 1, 3), (1, 3, 1), (3, 1, 1)):
    for _m in FWD_MODES:
        FWD_ROWS["k%d%d%d-%s" % (*_k, _m)] = (32, 48, _k, BASE, _m)
FWD_ROWS["lrelu_nostats"] = (32, 32, K3, BASE, "lrelu_nostats")
FWD_ROWS["d1_raw"] = (32, 64, K3, (2, 1, 20, 12), "bias")

WG_ROWS = {        # name: (Cin, Cout, k, (B, D, H, W)); the comment names the consumers the jobs run
    "ci16_k111": (16, 16, (1, 1, 1), (2, 3, 20, 12)),        # (16,1)
    "ci16_k113": (16, 72, (1, 1, 3), (1, 3, 20, 12)),        # (16,3)
    "ci16_k333": (16, 136, K3, (2, 3, 20, 12)),              # (16,9)
    "ci32_k311": (32, 48, (3, 1, 1), (1, 3, 20, 12)),        # (32,1)
    "ci32_k131": (32, 200, (1, 3, 1), (2, 3, 20, 12)),       # (32,3)
    "ci32_k333": (32, 128, K3, (1, 3, 20, 12)),              # (32,5) (32,4)
    "ci48_k111": (48, 72, (1, 1, 1), (2, 3, 20, 12)),        # (48,1)
    "ci48_k333": (48, 48, K3, (2, 3, 20, 12)),               # (48,3)
    "ci64_k111": (64, 136, (1, 1, 1), (1, 3, 20, 12)),       # (64,1)
    "ci64_k333": (64, 16, K3, (2, 3, 20, 12)),               # (64,3)
    "ci80_k333": (80, 200, K3, (1, 3, 20, 12)),              # (80,2) (80,1)
    "ci96_k333": (96, 72, K3, (2, 3, 20, 12)),               # (96,2) (96,1)
    "ci112_k133": (112, 128, (1, 3, 3), (1, 3, 20, 12)),     # (112,1)
    # several Cin tiles
    "ci176_k333": (176, 48, K3, (1, 3, 20, 12)),             # NTC 16
    "ci160_k333": (160, 136, K3, (2, 3, 20, 12)),            # NTC 32
    "ci240_k333": (240, 72, K3, (1, 3, 20, 12)),             # NTC 48
    "ci256_k333": (256, 200, K3, (1, 3, 20, 12)),            # NTC 64
    "ci192_k333": (192, 16, K3, (2, 3, 20, 12)),             # NTC 96
}
WG_ACTS = {"none": ACT_NONE, "relu": ACT_RELU, "lrelu": ACT_LRELU}

WG_EDGE_ROWS = {   # name: (Cin, Cout, k, (B, D, H, W), split-K factor S the row is there for)
    "s1_jobs144": (256, 512, K3, (1, 2, 16, 8), 1),           # 4 co x 4 ci tiles x 3 zd x 3 groups = 144 jobs >= 132
    "s1_one_tile_d1": (32, 64, K3, (1, 1, 16, 8), 1),         # one voxel tile; zd = 0 / 2 jobs own no valid tile
    "split_d1": (32, 64, K3, (2, 1, 40, 24), 18),             # S > 1 with D = 1, kd = 3: whole jobs store zero slices
    "split": (64, 128, K3, (2, 3, 20, 12), 14),
}
WG_BIAS_ROWS = {   # ALGO_AUTO with a bias gradient: column-sum pass + tensor-core weight gradient
    "split": (48, 144, (1, 1, 1), (1, 8, 16, 16), 16),
    "s1": (768, 3072, (1, 1, 1), (1, 4, 4, 4), 1),
}


# ----------------------------------------------------------------------------- CPU: the tables cover the library
def test_tables_reach_every_instantiation():
    cins = couts = range(16, 1025, 16)
    fwd_all = {fwd_inst(ci, co) for ci in cins for co in couts if tc_pick_nt(co)}
    assert len(fwd_all) == 32
    have = {}
    for ci, co, k, shape, mode in FWD_ROWS.values():
        have.setdefault(fwd_inst(ci, co), set()).add(mode)
    assert set(have) == fwd_all
    assert all(have[i] >= set(FWD_MODES) for i in fwd_all), {i: set(FWD_MODES) - have[i] for i in fwd_all}
    ntiles = {tc_pick_nt(co) for ci, co, *_ in FWD_ROWS.values() if tc_pick_nt(co) < co}
    nkc = {tc_pick_kc(ci) // 16 for ci, co, *_ in FWD_ROWS.values() if tc_pick_kc(ci) < ci and ci > 64}
    assert ntiles == set(NTS) and nkc == {1, 2, 3, 4}

    kernels = [(kd, kh, kw) for kd in (1, 3) for kh in (1, 3) for kw in (1, 3)]
    wg_all = set().union(*(wg_plan(ci, 64, k, (1, 1, 16, 8))[0] for ci in cins for k in kernels))
    assert len(wg_all) == 16
    wg_have = set().union(*(wg_plan(*r)[0] for r in WG_ROWS.values()))
    assert wg_have == wg_all
    assert {16, 48, 72, 128, 136, 200} <= {r[1] for r in WG_ROWS.values()}
    assert {ci // pick_ntc(ci) > 1 for ci, *_ in WG_ROWS.values()} == {False, True}


@pytest.fixture(scope="module")
def host_lib():
    import os
    from b200seg import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from b200seg.build import build
        build()
    return _lib.load()


def test_split_k_mirror_matches_library(host_lib):
    """the mirror's split-K factor S, as workspace bytes, is what b200seg_conv3d_wgrad_workspace reports"""
    from b200seg import _lib
    rows = [r[:4] for r in WG_ROWS.values()] + [r[:4] for r in WG_EDGE_ROWS.values()] + [r[:4] for r in WG_BIAS_ROWS.values()]
    for ci, co, k, shape in rows + [(c[0], c[1], c[2], c[3]) for c in WCASES]:
        _, S = wg_plan(ci, co, k, shape)
        want = S * co * ci * k[0] * k[1] * k[2] * 4 if S > 1 else 0
        got = host_lib.b200seg_conv3d_wgrad_workspace(ci, 0, 1, co, 0, 0, *shape, ci, co, *k, _lib.F16, _lib.ALGO_TC)
        assert got == want, (ci, co, k, shape, S)
    for ci, co, k, shape, S in list(WG_EDGE_ROWS.values()) + list(WG_BIAS_ROWS.values()):
        assert wg_plan(ci, co, k, shape)[1] == S


# ----------------------------------------------------------------------------- references
def randh(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def randf(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def seed_of(name):
    return zlib.crc32(name.encode()) & 0x7fffffff


def nc(t):
    """[B, D, H, W, C] -> float64 [B, C, D, H, W] on the device"""
    return t.double().permute(0, 4, 1, 2, 3)


def stats64(t):
    """InstanceNorm sums [B, C, 2] (fp64) of the stored values"""
    d = t.double().flatten(1, 3)
    return torch.stack([d.sum(1), (d * d).sum(1)], -1).contiguous()


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


def loader64(x, xst, act):
    """what the loaders stage: x itself, or fp16(act(IN(x))) (mean 0, rstd 1 without statistics)"""
    if xst is None and act == ACT_NONE:
        return nc(x)
    h = xhat64(x, xst) if xst is not None else nc(x)
    return act64(h, act).half().double()


def conv64(a, w16, k, bias=None):
    return F.conv3d(a, w16.double(), None if bias is None else bias.double(), padding=[i // 2 for i in k])


# ----------------------------------------------------------------------------- forward / data gradient
def _fwd_inputs(Cin, Cout, k, shape, mode, seed):
    B, D, H, W = shape
    taps = k[0] * k[1] * k[2]
    x = randh(B, D, H, W, Cin, seed=seed)
    w = randf(Cout, Cin, *k, seed=seed + 1) / (Cin * taps) ** 0.5
    inp = dict(x=x, w=w, xst=None, act=ACT_NONE, bias=None, res=None, dg=None, want_stats=True)
    if mode == "bias":
        inp.update(bias=randf(Cout, seed=seed + 2, scale=0.5), want_stats=False)
    elif mode in ("relu_res", "lrelu", "relu"):
        inp.update(xst=stats64(x), act=ACT_LRELU if mode == "lrelu" else ACT_RELU)
        if mode == "relu_res":
            inp["res"] = randh(B, D, H, W, Cout, seed=seed + 3)
    elif mode == "lrelu_nostats":
        inp["act"] = ACT_LRELU
    elif mode.startswith("dgrad"):
        gx = randh(B, D, H, W, Cout, seed=seed + 4)
        inp["dg"] = (gx, 0, stats64(gx), ACT_LRELU if mode == "dgrad_lrelu" else ACT_RELU)
    else:
        assert mode == "plain", mode
    return inp


def _fwd_ref(inp, k, act=None, g_act=None):
    """float64 forward of the launch described by inp (act / g_act override the activations: the ReLU twin of a
    LeakyReLU row); returns (ref, mask of the elements the bar applies to, pre-activation h of the dgrad mask or None)"""
    act = inp["act"] if act is None else act
    y = conv64(loader64(inp["x"], inp["xst"], act), inp["w"].half(), k, inp["bias"])
    if inp["res"] is not None:
        y = y.half().double() + nc(inp["res"])
    if inp["dg"] is None:
        return y, torch.ones_like(y, dtype=torch.bool), None
    gx, _, gst, ga = inp["dg"]
    h = xhat64(gx, gst)
    return y * dact64(h, ga if g_act is None else g_act), h.abs() >= MASK_MARGIN, h


def _masked_err(y, ref, keep):
    return rel_err(torch.where(keep, y, 0.0), torch.where(keep, ref, 0.0))


def _fwd_launch(inp, Cin, Cout, k, algo):
    from b200seg import ops
    wp = ops.pack_weight(inp["w"], torch.float16, layout=algo)
    return ops.conv3d_fwd(inp["x"], 0, Cin, inp["xst"], inp["act"], wp, Cout, k, bias=inp["bias"], residual=inp["res"],
                          want_stats=inp["want_stats"], dgrad_of=inp["dg"], algo=algo)


def _check_fwd(Cin, Cout, k, shape, mode, seed, record, direct=False):
    from b200seg import ops, _lib
    B = shape[0]
    assert ops.conv_algo(Cin, Cout, k, torch.float16, B) == _lib.ALGO_TC
    inp = _fwd_inputs(Cin, Cout, k, shape, mode, seed)
    yt, stt = _fwd_launch(inp, Cin, Cout, k, _lib.ALGO_TC)
    if direct:           # the CUDA-core kernel: same rounding model, different summation order
        yd, sd = _fwd_launch(inp, Cin, Cout, k, _lib.ALGO_DIRECT)
        assert rel_err(yt.float(), yd.float()) < 3e-3
        assert rel_err(stt, sd) < 1e-3
    torch.cuda.synchronize()
    ref, keep, h = _fwd_ref(inp, k)
    y = nc(yt)
    err = _masked_err(y, ref, keep)
    record("fwd_err", err)
    assert err < FWD_BAR, err
    if inp["act"] == ACT_LRELU or (inp["dg"] is not None and inp["dg"][3] == ACT_LRELU):
        twin, _, _ = _fwd_ref(inp, k, act=ACT_RELU if inp["act"] == ACT_LRELU else None, g_act=ACT_RELU)
        assert _masked_err(twin, ref, keep) > 3 * FWD_BAR, "this row cannot see the LeakyReLU slope"
    if not inp["want_stats"]:
        assert stt is None
        return
    if h is None:
        sref = stats64(yt)
    else:                # data-gradient mode: sum g and sum g * h of the stored g
        sref = torch.stack([y.sum((2, 3, 4)), (y * h).sum((2, 3, 4))], -1)
    serr = rel_err(stt, sref)
    record("stats_err", serr)
    assert serr < STATS_BAR, serr


@gpu
@pytest.mark.parametrize("row", list(FWD_ROWS))
def test_tc_fwd_matrix(row, record_property):
    Cin, Cout, k, shape, mode = FWD_ROWS[row]
    _check_fwd(Cin, Cout, k, shape, mode, seed_of(row), record_property)


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
CASE_MODES = {"plain": "plain", "norm": "relu", "normres": "relu_res", "dgrad": "dgrad_relu"}


@gpu
@pytest.mark.parametrize("Cin,Cout,k,shape,mode", CASES)
def test_tc_conv_matches_direct_and_torch(Cin, Cout, k, shape, mode, record_property):
    _check_fwd(Cin, Cout, k, shape, CASE_MODES[mode], 7, record_property, direct=True)


_INST = re.compile(r"conv_tc_kernel(?:<\s*(?:\(int\))?\s*(\d+)\s*,\s*(?:\(int\))?\s*(\d+)\s*>|ILi(\d+)ELi(\d+)E)")


@gpu
def test_every_conv_tc_instantiation_launches():
    """one base row per (NT, KSTEPS) under the profiler: the launched conv_tc_kernel<NT, KSTEPS> are all 32"""
    from torch.profiler import ProfilerActivity, profile
    from b200seg import _lib
    rows = {fwd_inst(r[0], r[1]): (name, r) for name, r in FWD_ROWS.items() if name.startswith("nt") and name.endswith("-bias")}
    assert len(rows) == 32
    launches = {}
    for inst, (name, (Cin, Cout, k, shape, mode)) in rows.items():
        launches[inst] = (_fwd_inputs(Cin, Cout, k, shape, mode, seed_of(name)), Cin, Cout, k)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
        for inp, Cin, Cout, k in launches.values():
            _fwd_launch(inp, Cin, Cout, k, _lib.ALGO_TC)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "conv_tc_kernel" in e.name}
    assert names, "the profiler recorded no conv_tc_kernel launch"
    seen = set()
    for n in names:
        m = _INST.search(n)
        assert m, n
        g = [int(v) for v in m.groups() if v is not None]
        seen.add((g[0], g[1]))
    print("conv_tc_kernel instantiations launched: %d of 32" % len(seen))
    assert seen == set(rows), sorted(set(rows) - seen)


# ----------------------------------------------------------------------------- weight gradient
def _wg_inputs(Cin, Cout, shape, act, seed):
    B, D, H, W = shape
    x = randh(B, D, H, W, Cin, seed=seed)
    dy = randh(B, D, H, W, Cout, seed=seed + 1)
    return x, (stats64(x) if act != ACT_NONE else None), dy


def _wg_ref(x, xst, act, dy, Cout, k, bias=False):
    a = loader64(x, xst, act)
    dw = torch.nn.grad.conv3d_weight(a, (Cout, a.shape[1], *k), nc(dy), padding=[i // 2 for i in k])
    return dw, (nc(dy).sum((0, 2, 3, 4)) if bias else None)


def wg_bar(act):
    return WG_BAR_RAW if act == ACT_NONE else WG_BAR


def _wg_slope_visible(x, xst, dy, Cout, k, ref):
    twin, _ = _wg_ref(x, xst, ACT_RELU, dy, Cout, k)
    assert rel_err(twin, ref) > 3 * WG_BAR, "this row cannot see the LeakyReLU slope"


@gpu
@pytest.mark.parametrize("act", list(WG_ACTS))
@pytest.mark.parametrize("row", list(WG_ROWS))
def test_tc_wgrad_matrix(row, act, record_property):
    from b200seg import ops, _lib
    Cin, Cout, k, shape = WG_ROWS[row]
    a = WG_ACTS[act]
    x, xst, dy = _wg_inputs(Cin, Cout, shape, a, seed_of(row + act))
    dw, _ = ops.conv3d_wgrad(x, 0, Cin, xst, a, dy, 0, Cout, k, algo=_lib.ALGO_TC)
    torch.cuda.synchronize()
    ref, _ = _wg_ref(x, xst, a, dy, Cout, k)
    err = rel_err(dw, ref)
    record_property("wg_err", err)
    assert err < wg_bar(a), err
    if a == ACT_LRELU:
        _wg_slope_visible(x, xst, dy, Cout, k, ref)


def _wgrad_raw(x, xst, act, dy, dw, db, k, algo):
    """b200seg_conv3d_wgrad into caller-provided dw / dbias (accumulated into, not zeroed)"""
    from b200seg import ops, _lib
    B, D, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    ws_bytes = _lib.load().b200seg_conv3d_wgrad_workspace(Cin, 0, 1 if (xst is not None or act) else 0, Cout, 0,
                                                          0 if db is None else 1, B, D, H, W, Cin, Cout, *k, _lib.F16, algo)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device="cuda")
    _lib.call("b200seg_conv3d_wgrad", x.data_ptr(), Cin, 0, None if xst is None else xst.data_ptr(), EPS, act,
              dy.data_ptr(), Cout, 0, dw.data_ptr(), None if db is None else db.data_ptr(),
              B, D, H, W, Cin, Cout, *k, _lib.F16, algo, ws.data_ptr(), ws_bytes, ops._stream())
    return ws_bytes


@gpu
@pytest.mark.parametrize("act", ["none", "lrelu"])
@pytest.mark.parametrize("row", list(WG_EDGE_ROWS))
def test_tc_wgrad_split_k_edges(row, act, record_property):
    """S == 1 (the CTA adds straight into dw) and S > 1 (slices summed in split order): the result is added to what dw
    holds, and a repeated call gives the same bits"""
    from b200seg import _lib
    Cin, Cout, k, shape, S = WG_EDGE_ROWS[row]
    a = WG_ACTS[act]
    x, xst, dy = _wg_inputs(Cin, Cout, shape, a, seed_of(row + act))
    prefill = randf(Cout, Cin, *k, seed=seed_of(row) + 5, scale=0.1)
    dw_acc = prefill.clone()
    ws_bytes = _wgrad_raw(x, xst, a, dy, dw_acc, None, k, _lib.ALGO_TC)
    assert (ws_bytes > 0) == (S > 1)
    runs = []
    for _ in range(2):
        runs.append(torch.zeros(Cout, Cin, *k, device="cuda"))
        _wgrad_raw(x, xst, a, dy, runs[-1], None, k, _lib.ALGO_TC)
    torch.cuda.synchronize()
    assert torch.equal(runs[0], runs[1])
    ref, _ = _wg_ref(x, xst, a, dy, Cout, k)
    err = max(rel_err(runs[0], ref), rel_err(dw_acc.double() - prefill.double(), ref))
    record_property("wg_err", err)
    assert err < wg_bar(a), err
    if a == ACT_LRELU:
        _wg_slope_visible(x, xst, dy, Cout, k, ref)


@gpu
@pytest.mark.parametrize("row", list(WG_BIAS_ROWS))
def test_tc_wgrad_bias_accumulates(row, record_property):
    """ALGO_AUTO with a bias gradient (column-sum pass + tensor cores) adds to non-zero dw and dbias"""
    from b200seg import _lib
    Cin, Cout, k, shape, S = WG_BIAS_ROWS[row]
    x, _, dy = _wg_inputs(Cin, Cout, shape, ACT_NONE, seed_of(row))
    dw0 = randf(Cout, Cin, *k, seed=seed_of(row) + 5, scale=0.1)
    db0 = randf(Cout, seed=seed_of(row) + 6, scale=10.0)
    dw, db = dw0.clone(), db0.clone()
    _wgrad_raw(x, None, ACT_NONE, dy, dw, db, k, _lib.ALGO_AUTO)
    runs = []
    for _ in range(2):
        runs.append((torch.zeros_like(dw), torch.zeros_like(db)))
        _wgrad_raw(x, None, ACT_NONE, dy, *runs[-1], k, _lib.ALGO_AUTO)
    torch.cuda.synchronize()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    wref, bref = _wg_ref(x, None, ACT_NONE, dy, Cout, k, bias=True)
    err = max(rel_err(runs[0][0], wref), rel_err(dw.double() - dw0.double(), wref))
    record_property("wg_err", err)
    assert err < WG_BAR_RAW, err
    assert rel_err(runs[0][1], bref) < 1e-5 and rel_err(db.double() - db0.double(), bref) < 1e-5


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


@gpu
@pytest.mark.parametrize("Cin,Cout,k,shape,normed", WCASES)
def test_tc_wgrad_matches_direct_and_torch(Cin, Cout, k, shape, normed, record_property):
    from b200seg import ops, _lib
    act = ACT_RELU if normed else ACT_NONE
    x, xst, dy = _wg_inputs(Cin, Cout, shape, act, 9)
    dwd, _ = ops.conv3d_wgrad(x, 0, Cin, xst, act, dy, 0, Cout, k, algo=_lib.ALGO_DIRECT)
    dwt, _ = ops.conv3d_wgrad(x, 0, Cin, xst, act, dy, 0, Cout, k, algo=_lib.ALGO_TC)
    assert rel_err(dwt, dwd) < 2e-3
    ref, _ = _wg_ref(x, xst, act, dy, Cout, k)
    err = rel_err(dwt, ref)
    record_property("wg_err", err)
    assert err < wg_bar(act), err


@gpu
@pytest.mark.parametrize("Cin,Cout,k,shape", [(48, 144, (1, 1, 1), (1, 8, 16, 16)),        # qkv Linear of SwinUNETR stage 1
                                              (192, 48, (1, 1, 1), (2, 4, 16, 8)),         # fc2
                                              (768, 3072, (1, 1, 1), (1, 4, 4, 4)),        # fc1 of the last stage: > 512 output channels
                                              (32, 24, (3, 3, 3), (1, 3, 16, 16))])
def test_biased_wgrad_takes_tensor_cores(Cin, Cout, k, shape, record_property):
    """A weight gradient WITH a bias gradient (every nn.Linear of SwinUNETR) = the column-sum pass + the tensor-core kernel
    (ALGO_AUTO), against the CUDA-core kernel that computes both (ALGO_DIRECT) and PyTorch float64."""
    from b200seg import ops, _lib
    x, _, dy = _wg_inputs(Cin, Cout, shape, ACT_NONE, 13)
    dwa, dba = ops.conv3d_wgrad(x, 0, Cin, None, ops.ACT_NONE, dy, 0, Cout, k, want_bias=True, algo=_lib.ALGO_AUTO)
    dwd, dbd = ops.conv3d_wgrad(x, 0, Cin, None, ops.ACT_NONE, dy, 0, Cout, k, want_bias=True, algo=_lib.ALGO_DIRECT)
    torch.cuda.synchronize()
    assert rel_err(dwa, dwd) < 2e-3 and rel_err(dba, dbd) < 2e-3
    wref, bref = _wg_ref(x, None, ACT_NONE, dy, Cout, k, bias=True)
    err = rel_err(dwa, wref)
    record_property("wg_err", err)
    assert err < WG_BAR_RAW and rel_err(dba, bref) < 1e-5, err
    assert not torch.equal(dwa, dwd)           # different kernels (split-K order), not the same code path twice
