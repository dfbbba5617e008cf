"""MedFormer-3D behind the reference's module contract (model/dim3/medformer.py:11-101, medformer_utils.py).

Same constructor arguments, the same module tree / parameter registration order, and therefore the same
`state_dict()` keys and shapes as the reference, so checkpoints, EMA zipping and DDP buckets are interchangeable
(SURVEY.md §8b).  The forward is written against libb200seg only: dense convs on the tensor-core path, depthwise convs,
B-MHA, map generation, SE, the token transformer — each a torch.autograd.Function from medformer_ops.py / ops.py.
Supported configuration = what the reference MedFormer YAMLs for BCV, AMOS, KiTS and ACDC use: norm 'in', act 'relu',
conv_block 'BasicBlock', proj_type 'depthwise', dropout 0, dim_head 32, 64 or 80 on attention levels, <= 80 map tokens,
and a map-fusion attention of dim_head 32 over <= 192 fused tokens or dim_head 64 over <= 216.  LiTS (one head of
128..320 channels) raises ValueError.
"""
import torch
import torch.nn as nn

from . import ops
from ._lib import ACT_NONE, ACT_RELU
from .medformer_ops import (AddFn, CatFn, ConvFn, DwConvFn, GeluFn, LayerNormFn, MHSAFn, MapGenFn, SEScaleFn,
                            SpaceToDepthFn, UpsampleFn)
from .ops import BiAttnFn, OutConvFn, PackedWeights, StemConvFn, UpCatFn
from .unet3d import BasicBlock, ConvNormAct, _check_kernel, _triple

EPS_BLOCK = 1e-4      # ConvNormAct's norm(in_ch, eps=1e-4), conv_layers.py:40
EPS_PLAIN = 1e-5      # bare norm(dim): PatchMerging.norm :158, BidirectionAttentionBlock.norm1/2 :107-108
BIATTN_DIM_HEADS = (32, 64, 80)     # csrc/biattn.cu: the original kernels (32, <= 64 tokens) and the wide ones
BIATTN_MAX_TOKENS = 80              # map tokens of B-MHA and map generation
MHSA_MAX_TOKENS = {32: 192, 64: 216}    # fused map tokens of the map-fusion attention per dim_head (b200seg_mhsa)


def _prod(size):
    n = 1
    for s in size:
        n *= int(s)
    return n


def _conv(pack, x, stats, weights, ksize, act=ACT_NONE, bias=None, residual=None, co_pad=0, eps=EPS_BLOCK,
          want_stats=False):
    """want_stats: produce the IN sums of the output (only when its consumer normalises it)."""
    packs = pack.get(list(weights), x.dtype, x.shape[0], co_pad)
    return ConvFn.apply(x, stats, residual, bias, packs, tuple(ksize), act, co_pad, eps, want_stats, *weights)


def _need_in(norm, act):
    if norm not in ('in', nn.InstanceNorm3d):
        raise ValueError("the H100 path implements InstanceNorm ('in') only, got norm=%r" % (norm,))
    if act not in ('relu', nn.ReLU):
        raise ValueError("the H100 path implements act='relu' only (every reference MedFormer config), got %r" % (act,))


class DepthwiseSeparableConv(nn.Module):
    """conv_layers.py:126-157."""

    def __init__(self, in_ch, out_ch, kernel_size=3):
        super().__init__()
        ks = _triple(kernel_size)
        _check_kernel(ks)
        pad = [i // 2 for i in ks]
        self.depthwise = nn.Conv3d(in_ch, in_ch, kernel_size=ks, padding=pad, groups=in_ch, bias=False)
        self.pointwise = nn.Conv3d(in_ch, out_ch, kernel_size=1, bias=False)
        self._pack = PackedWeights()

    def forward(self, x, stats, eps, residual=None, want_stats=False):
        """pointwise(depthwise(IN(x))) (+residual); stats=None means the input is used raw."""
        y, _ = DwConvFn.apply(x, stats, self.depthwise.weight, ACT_NONE, eps, False)
        return _conv(self._pack, y, None, [self.pointwise.weight], (1, 1, 1), residual=residual, want_stats=want_stats)


class BidirectionAttention(nn.Module):
    """medformer_utils.py:11-97."""

    def __init__(self, feat_dim, map_dim, out_dim, heads=4, dim_head=64, map_size=[8, 8, 8], proj_type='depthwise',
                 kernel_size=[3, 3, 3], no_map_out=False):
        super().__init__()
        if proj_type != 'depthwise':
            raise ValueError("the H100 path implements proj_type='depthwise' only")
        if dim_head not in BIATTN_DIM_HEADS:
            raise ValueError("the B-MHA kernels need dim_head in %s (got %d)" % (BIATTN_DIM_HEADS, dim_head))
        if _prod(map_size) > BIATTN_MAX_TOKENS:
            raise ValueError("the B-MHA kernels handle at most %d map tokens, got map_size=%s" % (BIATTN_MAX_TOKENS, map_size))
        self.inner_dim = dim_head * heads
        self.heads, self.dim_head = heads, dim_head
        self.feat_qv = DepthwiseSeparableConv(feat_dim, self.inner_dim * 2, kernel_size=kernel_size)
        self.feat_out = DepthwiseSeparableConv(self.inner_dim, out_dim, kernel_size=kernel_size)
        self.map_qv = nn.Conv3d(map_dim, self.inner_dim * 2, kernel_size=1, bias=False)
        self.map_out = nn.Identity() if no_map_out else nn.Conv3d(self.inner_dim, map_dim, kernel_size=1, bias=False)
        self._pack_mqv = PackedWeights()
        self._pack_mo = PackedWeights()

    def forward(self, x, x_stats, smap, feat_residual, map_residual):
        """x, smap raw (pre-norm) tensors; returns (feat_out + feat_residual, its sums, map_out + map_residual)."""
        fqv, _ = self.feat_qv(x, x_stats, EPS_PLAIN)                                       # :67
        m_stats = ops.instnorm_stats(smap, 0, smap.shape[-1])                              # norm2, :127
        mqv, _ = _conv(self._pack_mqv, smap, m_stats, [self.map_qv.weight], (1, 1, 1), eps=EPS_PLAIN)   # :68
        fo, mo = BiAttnFn.apply(fqv, mqv, self.heads, self.dim_head)                        # :70-91
        out, out_stats = self.feat_out(fo, None, EPS_PLAIN, residual=feat_residual, want_stats=True)   # :95 (+ :131)
        if isinstance(self.map_out, nn.Identity):
            mapp = AddFn.apply(mo, map_residual)
        else:
            mapp, _ = _conv(self._pack_mo, mo, None, [self.map_out.weight], (1, 1, 1), residual=map_residual)
        return out, out_stats, mapp


class SEBlock(nn.Module):
    """conv_layers.py:159-174."""

    def __init__(self, in_ch, ratio=4):
        super().__init__()
        self.squeeze = nn.AdaptiveAvgPool3d(1)
        self.excitation = nn.Sequential(nn.Conv3d(in_ch, in_ch // ratio, kernel_size=1), nn.ReLU(),
                                        nn.Conv3d(in_ch // ratio, in_ch, kernel_size=1), nn.Sigmoid())

    def forward(self, x, stats):
        e0, e2 = self.excitation[0], self.excitation[2]
        return SEScaleFn.apply(x, stats, e0.weight, e0.bias, e2.weight, e2.bias)


class MBConv(nn.Module):
    """conv_layers.py:197-238 with in_ch == out_ch, stride 1, se=True, p=0 (the only use in MedFormer)."""

    def __init__(self, in_ch, out_ch, expansion=4, kernel_size=3):
        super().__init__()
        if in_ch != out_ch or expansion == 1:
            raise ValueError("MBConv on the H100 path needs in_ch == out_ch and expansion > 1")
        ks = _triple(kernel_size)
        _check_kernel(ks)
        expanded = expansion * in_ch
        self.expand_proj = ConvNormAct(in_ch, expanded, kernel_size=1, padding=0)
        self.depthwise = nn.Module()          # ConvNormAct(groups=expanded): `conv` is its only stateful child
        self.depthwise.conv = nn.Conv3d(expanded, expanded, kernel_size=ks, padding=[(t - 1) // 2 for t in ks],
                                        groups=expanded, bias=False)
        self.se = SEBlock(expanded, ratio=4)
        self.pointwise = ConvNormAct(expanded, out_ch, kernel_size=1, padding=0)
        self.shortcut = nn.Sequential()
        self._pack_e = PackedWeights()
        self._pack_p = PackedWeights()

    def forward(self, x, stats):
        e, e_st = _conv(self._pack_e, x, stats, [self.expand_proj.conv.weight], (1, 1, 1), act=ACT_RELU, want_stats=True)  # :225
        d, d_st = DwConvFn.apply(e, e_st, self.depthwise.conv.weight, ACT_RELU, EPS_BLOCK, True)              # :226
        s, s_st = self.se(d, d_st)                                                                            # :228
        return _conv(self._pack_p, s, s_st, [self.pointwise.conv.weight], (1, 1, 1), act=ACT_NONE, residual=x,
                     want_stats=True)                                                                     # :230-234


class BidirectionAttentionBlock(nn.Module):
    """medformer_utils.py:102-138."""

    def __init__(self, feat_dim, map_dim, out_dim, heads, dim_head, expansion=4, map_size=[8, 8, 8],
                 proj_type='depthwise', kernel_size=[3, 3, 3], no_map_out=False):
        super().__init__()
        self.norm1 = nn.InstanceNorm3d(feat_dim)
        self.norm2 = nn.InstanceNorm3d(map_dim)
        self.attn = BidirectionAttention(feat_dim, map_dim, out_dim, heads, dim_head, map_size=map_size,
                                         proj_type=proj_type, kernel_size=kernel_size, no_map_out=no_map_out)
        self.shortcut = nn.Sequential()
        if feat_dim != out_dim:
            self.shortcut = ConvNormAct(feat_dim, out_dim, 1, padding=0)
        self.feedforward = MBConv(out_dim, out_dim, expansion=expansion, kernel_size=kernel_size)
        self._pack_sc = PackedWeights()

    def forward(self, x, x_stats, smap):
        if isinstance(self.shortcut, ConvNormAct):
            res, _ = _conv(self._pack_sc, x, x_stats, [self.shortcut.conv.weight], (1, 1, 1), act=ACT_RELU)   # :131
        else:
            res = x
        out, out_st, mapp = self.attn(x, x_stats, smap, res, smap)                                            # :129-136
        out, out_st = self.feedforward(out, out_st)                                                           # :132
        return out, out_st, mapp


class PatchMerging(nn.Module):
    """medformer_utils.py:140-177."""

    def __init__(self, dim, out_dim, proj_type='depthwise', down_scale=[2, 2, 2], kernel_size=[3, 3, 3]):
        super().__init__()
        if proj_type != 'depthwise':
            raise ValueError("the H100 path implements proj_type='depthwise' only")
        self.down_scale = tuple(int(s) for s in down_scale)
        merged_dim = 2 ** list(down_scale).count(2) * dim
        self.reduction = DepthwiseSeparableConv(merged_dim, out_dim, kernel_size=kernel_size)
        self.norm = nn.InstanceNorm3d(merged_dim)

    def forward(self, x):
        y, y_st = SpaceToDepthFn.apply(x, self.down_scale)            # :164-172
        return self.reduction(y, y_st, EPS_PLAIN, want_stats=True)    # :173-174


class BasicLayer(nn.Module):
    """medformer_utils.py:179-201."""

    def __init__(self, feat_dim, map_dim, out_dim, num_blocks, heads=4, dim_head=64, expansion=4, map_size=[8, 8, 8],
                 proj_type='depthwise', kernel_size=[3, 3, 3], no_map_out=False):
        super().__init__()
        dim1 = feat_dim
        self.blocks = nn.ModuleList([])
        for i in range(num_blocks):
            nmo = False if i != (num_blocks - 1) else no_map_out
            self.blocks.append(BidirectionAttentionBlock(dim1, map_dim, out_dim, heads, dim_head, expansion=expansion,
                                                         map_size=map_size, proj_type=proj_type,
                                                         kernel_size=kernel_size, no_map_out=nmo))
            dim1 = out_dim

    def forward(self, x, x_stats, smap):
        for block in self.blocks:
            x, x_stats, smap = block(x, x_stats, smap)
        return x, x_stats, smap


class SemanticMapGeneration(nn.Module):
    """medformer_utils.py:204-228.  base_proj and semantic_proj share their (raw) input: one GEMM, the map codes
    padded to a multiple of 16 output channels so the tensor-core path applies."""

    def __init__(self, feat_dim, map_dim, map_size):
        super().__init__()
        self.map_size = tuple(map_size)
        self.map_dim = map_dim
        self.map_code_num = map_size[0] * map_size[1] * map_size[2]
        if self.map_code_num > BIATTN_MAX_TOKENS:
            raise ValueError("the map kernels handle at most %d map tokens, got map_size=%s" % (BIATTN_MAX_TOKENS, map_size))
        self.base_proj = nn.Conv3d(feat_dim, map_dim, kernel_size=3, padding=1, bias=False)
        self.semantic_proj = nn.Conv3d(feat_dim, self.map_code_num, kernel_size=3, padding=1, bias=False)
        self._pack = PackedWeights()

    def forward(self, x):
        K = self.map_code_num
        pad = (-(self.map_dim + K)) % 16
        fw, _ = _conv(self._pack, x, None, [self.base_proj.weight, self.semantic_proj.weight], (3, 3, 3), co_pad=pad)
        return MapGenFn.apply(fw, self.map_dim, K, self.map_size)


class _Linear(nn.Linear):
    """nn.Linear evaluated as a 1x1x1 conv over tokens laid out [B,1,1,L,C]."""

    def run(self, pack, x, residual=None):
        w = self.weight.view(self.out_features, self.in_features, 1, 1, 1)
        y, _ = _conv(pack, x, None, [w], (1, 1, 1), bias=self.bias, residual=residual)
        return y


class Attention(nn.Module):
    """trans_layers.py:45-100."""

    def __init__(self, dim, heads, dim_head):
        super().__init__()
        if dim_head not in MHSA_MAX_TOKENS:
            raise ValueError("the token attention kernels need dim_head in %s (got %d)" % (tuple(MHSA_MAX_TOKENS), dim_head))
        self.heads, self.dim_head = heads, dim_head
        inner = dim_head * heads
        self.to_qkv = _Linear(dim, inner * 3, bias=False)
        self.to_out = _Linear(inner, dim)
        self._p1, self._p2 = PackedWeights(), PackedWeights()

    def forward(self, xn, residual):
        qkv = self.to_qkv.run(self._p1, xn)
        B, _, _, L, _ = qkv.shape
        att = MHSAFn.apply(qkv.view(B, L, -1), self.heads, self.dim_head)
        return self.to_out.run(self._p2, att.view(B, 1, 1, L, -1), residual=residual)


class Mlp(nn.Module):
    """trans_layers.py:16-33."""

    def __init__(self, in_dim, hid_dim=None, out_dim=None):
        super().__init__()
        self.fc1 = _Linear(in_dim, hid_dim or in_dim)
        self.act = nn.GELU()
        self.fc2 = _Linear(hid_dim or in_dim, out_dim or in_dim)
        self._p1, self._p2 = PackedWeights(), PackedWeights()

    def forward(self, xn, residual):
        h = GeluFn.apply(self.fc1.run(self._p1, xn))
        return self.fc2.run(self._p2, h, residual=residual)


class PreNorm(nn.Module):
    """trans_layers.py:35-41; the residual add of TransformerBlock (:113-114) rides in the last linear's epilogue."""

    def __init__(self, dim, fn):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.fn = fn

    def forward(self, x):
        xn = LayerNormFn.apply(x, self.norm.weight, self.norm.bias, self.norm.eps)
        return self.fn(xn, x)


class TransformerBlock(nn.Module):
    """trans_layers.py:103-118."""

    def __init__(self, dim, depth, heads, dim_head, mlp_dim):
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([PreNorm(dim, Attention(dim, heads, dim_head)),
                                              PreNorm(dim, Mlp(dim, mlp_dim, dim))]))

    def forward(self, x):
        for attn, ffn in self.layers:
            x = attn(x)
            x = ffn(x)
        return x


class SemanticMapFusion(nn.Module):
    """medformer_utils.py:231-268.  In channels-last the [B,C,d,h,w] -> [B,L,C] relayouts are views."""

    def __init__(self, in_dim_list, dim, heads, depth=1):
        super().__init__()
        self.dim = dim
        self.in_proj = nn.ModuleList([nn.Conv3d(c, dim, kernel_size=1, bias=False) for c in in_dim_list])
        self.fusion = TransformerBlock(dim, depth, heads, dim // heads, dim)
        self.out_proj = nn.ModuleList([nn.Conv3d(dim, c, kernel_size=1, bias=False) for c in in_dim_list])
        self._pi = [PackedWeights() for _ in in_dim_list]
        self._po = [PackedWeights() for _ in in_dim_list]

    def forward(self, map_list):
        B, md, mh, mw, _ = map_list[0].shape
        L = md * mh * mw
        toks = [_conv(self._pi[i], m, None, [self.in_proj[i].weight], (1, 1, 1))[0].view(B, L, self.dim)
                for i, m in enumerate(map_list)]
        x = torch.cat(toks, dim=1).view(B, 1, 1, L * len(map_list), self.dim)                # :258 (a copy, 81 tokens)
        x = self.fusion(x).view(B, L * len(map_list), self.dim)
        outs = []
        for i in range(len(map_list)):
            t = x[:, i * L:(i + 1) * L].contiguous().view(B, md, mh, mw, self.dim)          # :261
            outs.append(_conv(self._po[i], t, None, [self.out_proj[i].weight], (1, 1, 1))[0])
        return outs


class inconv(nn.Module):
    """medformer_utils.py:271-284."""

    def __init__(self, in_ch, out_ch, kernel_size=[3, 3, 3]):
        super().__init__()
        ks = _triple(kernel_size)
        _check_kernel(ks)
        self.ksize = tuple(ks)
        self.conv1 = nn.Conv3d(in_ch, out_ch, kernel_size=ks, padding=[i // 2 for i in ks], bias=False)
        self.conv2 = BasicBlock(out_ch, out_ch, kernel_size=ks)
        self._pack = PackedWeights()

    def forward(self, x):
        w = self.conv1.weight
        wf, _ = self._pack.get([w], x.dtype, x.shape[0])
        y, st = StemConvFn.apply(x, w, wf, self.ksize)
        return self.conv2((y, st))


class down_block(nn.Module):
    """medformer_utils.py:288-327."""

    def __init__(self, in_ch, out_ch, conv_num, trans_num, down_scale=[2, 2, 2], kernel_size=[3, 3, 3], heads=4,
                 dim_head=64, expansion=1, map_size=[8, 8, 8], proj_type='depthwise', map_generate=False, map_dim=None):
        super().__init__()
        map_dim = out_ch if map_dim is None else map_dim
        self.map_generate = map_generate
        if map_generate:
            self.map_gen = SemanticMapGeneration(out_ch, map_dim, map_size)
        self.patch_merging = PatchMerging(in_ch, out_ch, proj_type=proj_type, down_scale=down_scale, kernel_size=kernel_size)
        self.conv_blocks = nn.Sequential(*[BasicBlock(out_ch, out_ch, kernel_size=kernel_size) for _ in range(conv_num)])
        if trans_num and dim_head not in BIATTN_DIM_HEADS:
            raise ValueError("attention levels need dim_head in %s (got %d)" % (BIATTN_DIM_HEADS, dim_head))
        self.trans_blocks = BasicLayer(out_ch, map_dim, out_ch, num_blocks=trans_num, heads=heads,
                                       dim_head=dim_head if trans_num else 32, expansion=expansion, map_size=map_size,
                                       proj_type=proj_type, kernel_size=kernel_size)

    def forward(self, a):
        x, _ = a
        out = self.patch_merging(x)
        out = self.conv_blocks(out)
        smap = self.map_gen(out[0]) if self.map_generate else None
        y, y_st, smap = self.trans_blocks(out[0], out[1], smap)
        return (y, y_st), smap


class up_block(nn.Module):
    """medformer_utils.py:329-383."""

    def __init__(self, in_ch, out_ch, conv_num, trans_num, up_scale=[2, 2, 2], kernel_size=[3, 3, 3], heads=4,
                 dim_head=64, expansion=4, map_size=[4, 8, 8], proj_type='depthwise', map_dim=None, map_shortcut=False,
                 no_map_out=False):
        super().__init__()
        self.map_shortcut = map_shortcut
        map_dim = out_ch if map_dim is None else map_dim
        self.map_reduction = nn.Conv3d(in_ch + out_ch, map_dim, kernel_size=1, bias=False) if map_shortcut else nn.Identity()
        self.trans_blocks = BasicLayer(in_ch + out_ch, map_dim, out_ch, num_blocks=trans_num, heads=heads,
                                       dim_head=dim_head if trans_num else 32, expansion=expansion, map_size=map_size,
                                       proj_type=proj_type, kernel_size=kernel_size, no_map_out=no_map_out)
        dim1 = in_ch + out_ch if trans_num == 0 else out_ch
        blocks = []
        for _ in range(conv_num):
            blocks.append(BasicBlock(dim1, out_ch, kernel_size=kernel_size))
            dim1 = out_ch
        self.conv_blocks = nn.Sequential(*blocks)
        self._pack = PackedWeights()

    def forward(self, a1, a2, map1, map2=None):
        low, _ = a1
        skip, skip_st = a2
        feat, feat_st = UpCatFn.apply(low, skip, skip_st, False)                    # :386-387, order [up, skip]
        if self.map_shortcut and map2 is not None:
            smap, _ = _conv(self._pack, CatFn.apply(map1, map2), None, [self.map_reduction.weight], (1, 1, 1))  # :390-391
        else:
            smap = map1
        out, out_st, smap = self.trans_blocks(feat, feat_st, smap)
        out = self.conv_blocks((out, out_st))
        return out, smap


class MedFormer(nn.Module):
    """model/dim3/medformer.py:11-101 (constructor signature identical)."""

    def __init__(self, in_chan, num_classes, base_chan=32, map_size=[4, 8, 8], conv_block='BasicBlock',
                 conv_num=[2, 1, 0, 0, 0, 1, 2, 2], trans_num=[0, 1, 2, 2, 2, 1, 0, 0],
                 chan_num=[64, 128, 256, 320, 256, 128, 64, 32], num_heads=[1, 4, 8, 16, 8, 4, 1, 1], fusion_depth=2,
                 fusion_dim=320, fusion_heads=4, expansion=4, attn_drop=0., proj_drop=0., proj_type='depthwise',
                 norm='in', act='relu', kernel_size=[3, 3, 3, 3], scale=[2, 2, 2, 2], aux_loss=False):
        super().__init__()
        _need_in(norm, act)
        if conv_block not in ('BasicBlock', BasicBlock):
            raise ValueError("b200seg.MedFormer implements conv_block='BasicBlock' only")
        if attn_drop or proj_drop:
            raise ValueError("dropout is not implemented on the H100 path (every reference config uses 0)")
        dim_head = [chan_num[i] // num_heads[i] for i in range(8)]
        ks = [_triple(k) for k in kernel_size]
        sc = [_triple(s) for s in scale]
        common = dict(expansion=expansion, map_size=map_size, proj_type=proj_type)
        self.inc = inconv(in_chan, base_chan, kernel_size=ks[0])
        self.down1 = down_block(base_chan, chan_num[0], conv_num[0], trans_num[0], kernel_size=ks[1], down_scale=sc[0],
                                map_generate=False)
        self.down2 = down_block(chan_num[0], chan_num[1], conv_num[1], trans_num[1], kernel_size=ks[2], down_scale=sc[1],
                                heads=num_heads[1], dim_head=dim_head[1], map_generate=True, **common)
        self.down3 = down_block(chan_num[1], chan_num[2], conv_num[2], trans_num[2], kernel_size=ks[3], down_scale=sc[2],
                                heads=num_heads[2], dim_head=dim_head[2], map_generate=True, **common)
        self.down4 = down_block(chan_num[2], chan_num[3], conv_num[3], trans_num[3], kernel_size=ks[4], down_scale=sc[3],
                                heads=num_heads[3], dim_head=dim_head[3], map_generate=True, **common)
        fused, fdh = 3 * _prod(map_size), fusion_dim // fusion_heads
        if fdh in MHSA_MAX_TOKENS and fused > MHSA_MAX_TOKENS[fdh]:
            raise ValueError("the map-fusion attention at dim_head %d handles at most %d tokens, got 3 x %d"
                             % (fdh, MHSA_MAX_TOKENS[fdh], _prod(map_size)))
        self.map_fusion = SemanticMapFusion(chan_num[1:4], fusion_dim, fusion_heads, depth=fusion_depth)
        self.up1 = up_block(chan_num[3], chan_num[4], conv_num[4], trans_num[4], kernel_size=ks[3], up_scale=sc[3],
                            heads=num_heads[4], dim_head=dim_head[4], map_shortcut=True, **common)
        self.up2 = up_block(chan_num[4], chan_num[5], conv_num[5], trans_num[5], kernel_size=ks[2], up_scale=sc[2],
                            heads=num_heads[5], dim_head=dim_head[5], map_shortcut=True, no_map_out=True, **common)
        self.up3 = up_block(chan_num[5], chan_num[6], conv_num[6], trans_num[6], kernel_size=ks[1], up_scale=sc[1],
                            map_shortcut=False)
        self.up4 = up_block(chan_num[6], chan_num[7], conv_num[7], trans_num[7], kernel_size=ks[0], up_scale=sc[0],
                            map_shortcut=False)
        self.aux_loss = aux_loss
        if aux_loss:
            self.aux_out = nn.Conv3d(chan_num[5], num_classes, kernel_size=1)
        self.outc = nn.Conv3d(chan_num[7], num_classes, kernel_size=1)
        self.num_classes = num_classes
        self._pack_out, self._pack_aux = PackedWeights(), PackedWeights()
        self._packs = ops.PackRegistry(self)

    def forward(self, x):
        if not x.is_cuda:
            raise ops._lib.B200SegError("b200seg.MedFormer runs on an H100 only — there is no CPU fallback")
        with ops.on_device(x):
            return self._forward(x)

    def _forward(self, x):
        dt = ops.compute_dtype()
        self._packs.refresh()           # every packed weight image is rebuilt from the live parameters (one launch)
        xin = x.permute(0, 2, 3, 4, 1).to(dt).contiguous()
        x0 = self.inc(xin)
        x1, _ = self.down1(x0)
        x2, map2 = self.down2(x1)
        x3, map3 = self.down3(x2)
        x4, map4 = self.down4(x3)
        maps = self.map_fusion([map2, map3, map4])
        out, smap = self.up1(x4, x3, maps[2], maps[1])
        out, smap = self.up2(out, x2, smap, maps[0])
        aux = None
        if self.aux_loss:
            pad = (-self.num_classes) % 8
            a, _ = _conv(self._pack_aux, out[0], None, [self.aux_out.weight], (1, 1, 1), bias=self.aux_out.bias, co_pad=pad)
            a = UpsampleFn.apply(a, tuple(xin.shape[1:4]))
            aux = a[..., :self.num_classes].permute(0, 4, 1, 2, 3)
        out, smap = self.up3(out, x1, smap, None)
        out, smap = self.up4(out, x0, smap, None)
        w, b = self.outc.weight, self.outc.bias
        logits = OutConvFn.apply(out[0], w, b, self._pack_out.get([w], dt, x.shape[0])).permute(0, 4, 1, 2, 3)
        return [logits, aux] if self.aux_loss else logits
