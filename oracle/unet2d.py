"""CPU restatement of the reference 2D UNet (model/dim2/unet.py with unet_utils.py and the SingleConv / BasicBlock of
conv_layers.py, BatchNorm2d + ReLU) and of its inference functions (inference/inference2d.py), in stock PyTorch.

Same module tree and state_dict keys as the reference class, so fixtures and state_dicts move between the two;
oracle/make_golden_unet2d.py pins it to the unmodified reference.  Test infrastructure and the stock-torch arm of
tools/unet2d_bench.py: the package never imports it."""
import torch
import torch.nn as nn
import torch.nn.functional as F


class ConvNormAct(nn.Module):
    def __init__(self, in_ch, out_ch, preact):
        super().__init__()
        self.conv = nn.Conv2d(in_ch, out_ch, 3, padding=1, bias=False)
        self.norm = nn.BatchNorm2d(in_ch if preact else out_ch)
        self.act = nn.ReLU()
        self.preact = preact

    def forward(self, x):
        if self.preact:
            return self.conv(self.act(self.norm(x)))
        return self.act(self.norm(self.conv(x)))


class SingleConv(nn.Module):
    def __init__(self, in_ch, out_ch):
        super().__init__()
        self.conv = ConvNormAct(in_ch, out_ch, preact=False)

    def forward(self, x):
        return self.conv(x)


class BasicBlock(nn.Module):
    def __init__(self, in_ch, out_ch):
        super().__init__()
        self.conv1 = ConvNormAct(in_ch, out_ch, preact=True)
        self.conv2 = ConvNormAct(out_ch, out_ch, preact=True)
        self.shortcut = ConvNormAct(in_ch, out_ch, preact=True) if in_ch != out_ch else nn.Sequential()

    def forward(self, x):
        return self.conv2(self.conv1(x)) + self.shortcut(x)


class inconv(nn.Module):
    def __init__(self, in_ch, out_ch, block):
        super().__init__()
        self.conv1 = nn.Conv2d(in_ch, out_ch, 3, padding=1, bias=False)
        self.conv2 = block(out_ch, out_ch)

    def forward(self, x):
        return self.conv2(self.conv1(x))


class down_block(nn.Module):
    def __init__(self, in_ch, out_ch, block):
        super().__init__()
        self.conv = nn.Sequential(nn.MaxPool2d(2), block(in_ch, out_ch), block(out_ch, out_ch))

    def forward(self, x):
        return self.conv(x)


class up_block(nn.Module):
    def __init__(self, in_ch, out_ch, block):
        super().__init__()
        self.conv_ch = nn.Conv2d(in_ch, out_ch, 1)
        self.conv = nn.Sequential(block(2 * out_ch, out_ch), block(out_ch, out_ch))

    def forward(self, x1, x2):
        x1 = self.conv_ch(F.interpolate(x1, scale_factor=2, mode="bilinear", align_corners=True))
        return self.conv(torch.cat([x2, x1], 1))


class UNet2DRef(nn.Module):
    def __init__(self, in_ch, num_classes, base_ch=32, block="SingleConv"):
        super().__init__()
        blk = {"SingleConv": SingleConv, "BasicBlock": BasicBlock}[block]
        self.inc = inconv(in_ch, base_ch, blk)
        self.down1 = down_block(base_ch, 2 * base_ch, blk)
        self.down2 = down_block(2 * base_ch, 4 * base_ch, blk)
        self.down3 = down_block(4 * base_ch, 8 * base_ch, blk)
        self.down4 = down_block(8 * base_ch, 16 * base_ch, blk)
        self.up1 = up_block(16 * base_ch, 8 * base_ch, blk)
        self.up2 = up_block(8 * base_ch, 4 * base_ch, blk)
        self.up3 = up_block(4 * base_ch, 2 * base_ch, blk)
        self.up4 = up_block(2 * base_ch, base_ch, blk)
        self.outc = nn.Conv2d(base_ch, num_classes, 1)

    def forward(self, x):
        x1 = self.inc(x)
        x2 = self.down1(x1)
        x3 = self.down2(x2)
        x4 = self.down3(x3)
        x5 = self.down4(x4)
        out = self.up4(self.up3(self.up2(self.up1(x5, x4), x3), x2), x1)
        return self.outc(out)


def _split_idx(half_win, size, i):
    start = half_win * i
    if start + 2 * half_win > size:
        start = size - 2 * half_win
    return start, start + 2 * half_win


def inference_whole_image(net, img, args=None):
    """inference/inference2d.py: softmax of one eval-mode forward of the whole slice batch."""
    net.eval()
    with torch.no_grad():
        pred = net(img)
    return F.softmax(pred, dim=1)


def inference_sliding_window(net, img, args):
    """inference/inference2d.py: half-window stride, last window snapped to the border, softmax averaged."""
    net.eval()
    B, C, H, W = img.shape
    win_h, win_w = args.window_size
    hh, hw = win_h // 2, win_w // 2
    out = torch.zeros(B, args.classes, H, W, device=img.device)
    counter = torch.zeros(B, 1, H, W, device=img.device)
    with torch.no_grad():
        for i in range(H // hh):
            for j in range(W // hw):
                h0, h1 = _split_idx(hh, H, i)
                w0, w1 = _split_idx(hw, W, j)
                out[:, :, h0:h1, w0:w1] += F.softmax(net(img[:, :, h0:h1, w0:w1]), dim=1)
                counter[:, :, h0:h1, w0:w1] += 1
    return out / counter
