"""2D UNet / ResUNet whose every op runs in libb200seg.so — drop-in for the reference's ``model/dim2/unet.py:7-43``
(+ ``unet_utils.py``, ``conv_layers.py:21-94``) with ``block='SingleConv'`` (``unet``) or ``'BasicBlock'``
(``resunet``), ``pool=True``: same constructor, module tree, ``state_dict`` keys / shapes / buffers, parameter
registration order and default initialisation.  The ``nn.Conv2d`` / ``nn.BatchNorm2d`` modules only hold state and are
never called; the BatchNorm holders are looked up at every forward, so ``nn.SyncBatchNorm.convert_sync_batchnorm``
may replace them and their momentum / eps are honoured.

Activations are NDHWC buffers with D = 1; a 3x3 Conv2d is a (1,3,3) convolution, MaxPool2d(2) is max-pool at (1,2,2)
and bilinear upsampling with align_corners=True is the trilinear kernel at (1,2,2).  ``up_block.conv_ch`` (1x1 with
bias) runs before the upsample instead of after it: the align_corners weights of each output pixel sum to 1, so the
result is the same in real arithmetic, the 1x1 touches a quarter of the pixels, and the upsample writes straight into
the concat buffer.
"""
import torch
import torch.nn as nn

from . import ops
from .batchnorm import BNBasicBlockFn, BNSingleConvFn, PointwiseConvFn
from .ops import MaxPoolFn, PackedWeights, StemConvFn, UpCatFn

K33 = (1, 3, 3)


def _w5(conv):
    """A Conv2d weight [Cout, Cin, kh, kw] as the (1, kh, kw) convolution weight the library takes (a view)."""
    w = conv.weight
    return w.view(w.shape[0], w.shape[1], 1, w.shape[2], w.shape[3])


class ConvNormAct(nn.Module):
    """Parameter holder mirroring conv_layers.py:21-53 with norm=nn.BatchNorm2d, act=nn.ReLU."""

    def __init__(self, in_ch, out_ch, kernel_size=3, padding=1, preact=False):
        super().__init__()
        self.conv = nn.Conv2d(in_ch, out_ch, kernel_size=kernel_size, padding=padding, bias=False)
        self.norm = nn.BatchNorm2d(in_ch if preact else out_ch)
        self.act = nn.ReLU()
        self.preact = preact


class SingleConv(nn.Module):
    """conv -> BN -> ReLU (conv_layers.py:56-68, post-activation)."""

    def __init__(self, in_ch, out_ch):
        super().__init__()
        self.conv = ConvNormAct(in_ch, out_ch, 3, padding=1, preact=False)
        self._pack = PackedWeights()

    def forward(self, a):
        x, _ = a
        w = _w5(self.conv.conv)
        bn = self.conv.norm
        y = BNSingleConvFn.apply(x, w, bn.weight, bn.bias, bn, self._pack.get([w], x.dtype, 1), K33)
        return (y, None)


class BasicBlock(nn.Module):
    """Pre-activation residual block (conv_layers.py:71-94)."""

    def __init__(self, in_ch, out_ch):
        super().__init__()
        self.conv1 = ConvNormAct(in_ch, out_ch, 3, padding=1, preact=True)
        self.conv2 = ConvNormAct(out_ch, out_ch, 3, padding=1, preact=True)
        self.shortcut = nn.Sequential()
        if in_ch != out_ch:
            self.shortcut = ConvNormAct(in_ch, out_ch, 3, padding=1, preact=True)
        self._pack_1 = PackedWeights()
        self._pack_2 = PackedWeights()
        self._pack_s = PackedWeights()

    def forward(self, a):
        x, xs = a
        if xs is None or xs.numel() == 0:
            xs = ops.instnorm_stats(x, 0, x.shape[-1])
        c1, c2 = self.conv1, self.conv2
        w1, w2 = _w5(c1.conv), _w5(c2.conv)
        dt = x.dtype
        packs = [self._pack_1.get([w1], dt, 1), self._pack_2.get([w2], dt, 1), None]
        if isinstance(self.shortcut, ConvNormAct):
            cs = self.shortcut
            ws, gs, bs, bn_s = _w5(cs.conv), cs.norm.weight, cs.norm.bias, cs.norm
            packs[2] = self._pack_s.get([ws], dt, 1)
        else:
            ws = gs = bs = bn_s = None
        out, out_sums = BNBasicBlockFn.apply(x, xs, w1, c1.norm.weight, c1.norm.bias, w2, c2.norm.weight, c2.norm.bias,
                                             ws, gs, bs, (c1.norm, c2.norm, bn_s), tuple(packs), K33)
        return (out, out_sums)


_BLOCKS = {"SingleConv": SingleConv, "BasicBlock": BasicBlock}


def get_block(name):
    """model/dim2/utils.py get_block, for the blocks of the ACDC 2D configs."""
    if name not in _BLOCKS:
        raise ValueError("2d block %r is not supported by the H100 path (have %s)" % (name, sorted(_BLOCKS)))
    return _BLOCKS[name]


class inconv(nn.Module):
    """unet_utils.py:7-18: raw 3x3 Conv2d stem, then one block."""

    def __init__(self, in_ch, out_ch, block=BasicBlock):
        super().__init__()
        self.conv1 = nn.Conv2d(in_ch, out_ch, kernel_size=3, padding=1, bias=False)
        self.conv2 = block(out_ch, out_ch)
        self._pack = PackedWeights()

    def forward(self, x):
        w = _w5(self.conv1)
        wf, _ = self._pack.get([w], x.dtype, 1)
        y, st = StemConvFn.apply(x, w, wf, K33)
        return self.conv2((y, st))


class _Pool(nn.Module):
    """Stands in index 0 of down_block.conv (nn.MaxPool2d(2), no state) so block indices match the reference."""

    def forward(self, a):
        x, _ = a
        return MaxPoolFn.apply(x, (1, 2, 2), True)


class down_block(nn.Module):
    """unet_utils.py:21-38 with pool=True."""

    def __init__(self, in_ch, out_ch, num_block, block=BasicBlock, pool=True):
        super().__init__()
        if not pool:
            raise ValueError("pool=False (strided conv downsampling) is not supported by the H100 path")
        layers = [_Pool(), block(in_ch, out_ch)]
        for _ in range(num_block - 1):
            layers.append(block(out_ch, out_ch))
        self.conv = nn.Sequential(*layers)

    def forward(self, a):
        return self.conv(a)


class up_block(nn.Module):
    """unet_utils.py:40-61: bilinear x2 (align_corners=True), conv_ch (1x1 with bias), cat([skip, up]), blocks."""

    def __init__(self, in_ch, out_ch, num_block, block=BasicBlock):
        super().__init__()
        self.conv_ch = nn.Conv2d(in_ch, out_ch, kernel_size=1)
        layers = [block(2 * out_ch, out_ch)]
        for _ in range(num_block - 1):
            layers.append(block(out_ch, out_ch))
        self.conv = nn.Sequential(*layers)
        self._pack = PackedWeights()

    def forward(self, a1, a2):
        low, _ = a1
        skip, skip_sums = a2
        if skip.shape[2] != 2 * low.shape[2] or skip.shape[3] != 2 * low.shape[3]:
            raise ValueError("up_block expects the skip at twice the resolution (F.interpolate(scale_factor=2)); "
                             "got %s and %s" % (tuple(low.shape[1:4]), tuple(skip.shape[1:4])))
        w = _w5(self.conv_ch)
        low = PointwiseConvFn.apply(low, w, self.conv_ch.bias, self._pack.get([w], low.dtype, 1))
        cat, cat_sums = UpCatFn.apply(low, skip, skip_sums, True)
        return self.conv((cat, cat_sums))


class UNet2D(nn.Module):
    """model/dim2/unet.py:7-43 (``UNet(in_ch, num_classes, base_ch=32, block='SingleConv', pool=True)``)."""

    def __init__(self, in_ch, num_classes, base_ch=32, block='SingleConv', pool=True):
        super().__init__()
        blk = get_block(block)
        nb = 2
        self.inc = inconv(in_ch, base_ch, block=blk)
        self.down1 = down_block(base_ch, 2 * base_ch, num_block=nb, block=blk, pool=pool)
        self.down2 = down_block(2 * base_ch, 4 * base_ch, num_block=nb, block=blk, pool=pool)
        self.down3 = down_block(4 * base_ch, 8 * base_ch, num_block=nb, block=blk, pool=pool)
        self.down4 = down_block(8 * base_ch, 16 * base_ch, num_block=nb, block=blk, pool=pool)
        self.up1 = up_block(16 * base_ch, 8 * base_ch, num_block=nb, block=blk)
        self.up2 = up_block(8 * base_ch, 4 * base_ch, num_block=nb, block=blk)
        self.up3 = up_block(4 * base_ch, 2 * base_ch, num_block=nb, block=blk)
        self.up4 = up_block(2 * base_ch, base_ch, num_block=nb, block=blk)
        self.outc = nn.Conv2d(base_ch, num_classes, kernel_size=1)
        self._pack_out = PackedWeights()
        self._packs = ops.PackRegistry(self)

    def forward(self, x):
        if not x.is_cuda:
            raise ops._lib.B200SegError("b200seg.UNet2D runs on an H100 only — there is no CPU fallback")
        if x.dim() != 4:
            raise ValueError("UNet2D takes [B, C, H, W] input, got shape %s" % (tuple(x.shape),))
        with ops.on_device(x):
            return self._forward(x)

    def _forward(self, x):
        dt = ops.compute_dtype()
        self._packs.refresh()
        # boundary: NCHW input -> [B, 1, H, W, C] working layout (free when in_ch == 1)
        xin = x.permute(0, 2, 3, 1).unsqueeze(1).to(dt).contiguous()
        x1 = self.inc(xin)
        x2 = self.down1(x1)
        x3 = self.down2(x2)
        x4 = self.down3(x3)
        x5 = self.down4(x4)
        out = self.up1(x5, x4)
        out = self.up2(out, x3)
        out = self.up3(out, x2)
        out = self.up4(out, x1)
        w = _w5(self.outc)
        logits = PointwiseConvFn.apply(out[0], w, self.outc.bias, self._pack_out.get([w], dt, 1))
        # boundary: logical NCHW shape over the [B, 1, H, W, C] buffer (channels_last strides, zero-copy)
        return logits.squeeze(1).permute(0, 3, 1, 2)
