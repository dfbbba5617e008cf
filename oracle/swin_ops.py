"""ORACLE (test infrastructure — never imported by the product path).

CPU restatement of the Swin pieces that are VENDORED in the reference (model/dim3/swin_unetr.py) — the part of
SwinUNETR whose behaviour can be pinned here, because it does not live in the absent `monai` package:
  relative_position_index        WindowAttention.__init__   swin_unetr.py:417-459
  window_partition / reverse     swin_unetr.py:295-355
  get_window_size                swin_unetr.py:358-381
  compute_mask                   swin_unetr.py:737-773
  window_attention               WindowAttention.forward     swin_unetr.py:467-490
  swin_block_part1               SwinTransformerBlock.forward_part1  swin_unetr.py:554-606
  window_attention_core          forward_part1 between the qkv and proj Linears, chunked (the window-attention kernels' operator)
  patch_merging                  PatchMerging.forward (v0.9 ordering, with its duplicated slices)  swin_unetr.py:707-731
Pinned by oracle/make_golden_swin.py against the unmodified classes (imported with a throw-away stand-in for the
seven monai symbols the file pulls in) -> tests/golden/swin_*.pt.  The monai-defined blocks (MLPBlock, PatchEmbed,
UnetrBasicBlock, UnetrUpBlock, UnetOutBlock) are NOT restated here: their source is not under /root/reference
("parity unpinned" in SURVEY.md §8c).  No CUDA kernel consumes this yet — it is the round-2 starting point for rows
a15/a16.
"""
import itertools

import torch
import torch.nn.functional as F


def relative_position_index(window_size):
    """[n, n] int64 index into the (2w0-1)(2w1-1)(2w2-1) bias table — swin_unetr.py:424-441,459."""
    ws = list(window_size)
    coords = torch.stack(torch.meshgrid(*[torch.arange(s) for s in ws], indexing="ij"))
    flat = torch.flatten(coords, 1)
    rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws[0] - 1
    rel[:, :, 1] += ws[1] - 1
    rel[:, :, 2] += ws[2] - 1
    rel[:, :, 0] *= (2 * ws[1] - 1) * (2 * ws[2] - 1)
    rel[:, :, 1] *= 2 * ws[2] - 1
    return rel.sum(-1)


def window_partition(x, ws):
    """[b,d,h,w,c] -> [b*nW, ws0*ws1*ws2, c] — swin_unetr.py:305-320."""
    b, d, h, w, c = x.shape
    x = x.view(b, d // ws[0], ws[0], h // ws[1], ws[1], w // ws[2], ws[2], c)
    return x.permute(0, 1, 3, 5, 2, 4, 6, 7).contiguous().view(-1, ws[0] * ws[1] * ws[2], c)


def window_reverse(windows, ws, dims):
    """inverse of window_partition — swin_unetr.py:337-349."""
    b, d, h, w = dims
    x = windows.view(b, d // ws[0], h // ws[1], w // ws[2], ws[0], ws[1], ws[2], -1)
    return x.permute(0, 1, 4, 2, 5, 3, 6, 7).contiguous().view(b, d, h, w, -1)


def get_window_size(x_size, window_size, shift_size=None):
    """Clamp window (and zero the shift) on axes not larger than the window — swin_unetr.py:369-381."""
    use_w = list(window_size)
    use_s = list(shift_size) if shift_size is not None else None
    for i in range(len(x_size)):
        if x_size[i] <= window_size[i]:
            use_w[i] = x_size[i]
            if use_s is not None:
                use_s[i] = 0
    return tuple(use_w) if use_s is None else (tuple(use_w), tuple(use_s))


def compute_mask(dims, window_size, shift_size):
    """[nW, n, n] additive mask, 0 inside a region and -100 across regions — swin_unetr.py:750-773."""
    d, h, w = dims
    img = torch.zeros((1, d, h, w, 1))
    cnt = 0
    for sd in (slice(-window_size[0]), slice(-window_size[0], -shift_size[0]), slice(-shift_size[0], None)):
        for sh in (slice(-window_size[1]), slice(-window_size[1], -shift_size[1]), slice(-shift_size[1], None)):
            for sw in (slice(-window_size[2]), slice(-window_size[2], -shift_size[2]), slice(-shift_size[2], None)):
                img[:, sd, sh, sw, :] = cnt
                cnt += 1
    mw = window_partition(img, window_size).squeeze(-1)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def window_attention(x, p, heads, rel_index, mask=None):
    """x [b*nW, n, c]; p: dict(qkv_w, qkv_b|None, proj_w, proj_b, bias_table [T, heads]) — swin_unetr.py:467-490."""
    b, n, c = x.shape
    qkv = F.linear(x, p["qkv_w"], p.get("qkv_b")).reshape(b, n, 3, heads, c // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * (c // heads) ** -0.5, qkv[1], qkv[2]
    attn = q @ k.transpose(-2, -1)
    bias = p["bias_table"][rel_index[:n, :n].reshape(-1)].reshape(n, n, -1).permute(2, 0, 1)
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nw = mask.shape[0]
        attn = (attn.view(b // nw, nw, heads, n, n) + mask.unsqueeze(1).unsqueeze(0)).view(-1, heads, n, n)
    attn = F.softmax(attn, dim=-1).to(v.dtype)
    return F.linear((attn @ v).transpose(1, 2).reshape(b, n, c), p["proj_w"], p["proj_b"])


def swin_block_part1(x, p, heads, window_size, shift_size, mask_matrix):
    """LayerNorm, pad to a window multiple, cyclic shift, windowed attention, un-shift, crop — swin_unetr.py:554-606.
    x [b,d,h,w,c]; p additionally holds norm1_w / norm1_b."""
    b, d, h, w, c = x.shape
    x = F.layer_norm(x, (c,), p["norm1_w"], p["norm1_b"])
    ws, ss = get_window_size((d, h, w), window_size, shift_size)
    pad_d = (ws[0] - d % ws[0]) % ws[0]
    pad_b = (ws[1] - h % ws[1]) % ws[1]
    pad_r = (ws[2] - w % ws[2]) % ws[2]
    x = F.pad(x, (0, 0, 0, pad_r, 0, pad_b, 0, pad_d))
    _, dp, hp, wp, _ = x.shape
    shifted = any(i > 0 for i in ss)
    if shifted:
        x = torch.roll(x, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
    rel = relative_position_index(window_size)
    win = window_attention(window_partition(x, ws), p, heads, rel, mask_matrix if shifted else None)
    x = window_reverse(win.view(-1, *(ws + (c,))), ws, [b, dp, hp, wp])
    if shifted:
        x = torch.roll(x, shifts=(ss[0], ss[1], ss[2]), dims=(1, 2, 3))
    return x[:, :d, :h, :w, :].contiguous()


def _round16(t):
    """t rounded to fp16 in value, with an identity gradient (autocast rounds the forward value only)."""
    return t + (t.half().to(t.dtype) - t).detach()


def _attention_core(x, table, rel, mask, heads, fp16_rounding):
    """x [w, n, 3C] partitioned qkv windows -> [w, n, C]: the middle of WindowAttention.forward, swin_unetr.py:467-490.
    mask [w, n, n] or None."""
    w, n, c3 = x.shape
    c = c3 // 3
    qkv = x.reshape(w, n, 3, heads, c // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * (c // heads) ** -0.5, qkv[1], qkv[2]
    if fp16_rounding:
        q = _round16(q)                                      # autocast: `q * self.scale` is an fp16 tensor
    attn = q @ k.transpose(-2, -1) + table[rel.reshape(-1)].reshape(n, n, heads).permute(2, 0, 1).unsqueeze(0)
    if mask is not None:
        attn = attn + mask.unsqueeze(1)
    attn = F.softmax(attn, dim=-1)
    if fp16_rounding:
        attn = _round16(attn)                                # `attn.to(v.dtype)` before `@ v`
    return (attn @ v).transpose(1, 2).reshape(w, n, c)


class _ChunkedCore(torch.autograd.Function):
    """_attention_core over chunks of windows; the backward recomputes each chunk, so the [w, heads, n, n] scores of one
    chunk at a time are all that is ever held (stage 1 of a 128^3 SwinUNETR has 1000 windows of 343 tokens)."""

    @staticmethod
    def forward(ctx, xw, table, rel, mask, heads, fp16_rounding, chunk):
        ctx.save_for_backward(xw, table, rel, mask)
        ctx.meta = (heads, fp16_rounding, chunk)
        nw = 1 if mask is None else mask.shape[0]
        outs = []
        for i in range(0, xw.shape[0], chunk):
            j = min(i + chunk, xw.shape[0])
            m = None if mask is None else mask[torch.arange(i, j, device=xw.device) % nw]
            outs.append(_attention_core(xw[i:j], table, rel, m, heads, fp16_rounding))
        return torch.cat(outs)

    @staticmethod
    def backward(ctx, dout):
        xw, table, rel, mask = ctx.saved_tensors
        heads, fp16_rounding, chunk = ctx.meta
        nw = 1 if mask is None else mask.shape[0]
        dx, dt = torch.empty_like(xw), torch.zeros_like(table)
        for i in range(0, xw.shape[0], chunk):
            j = min(i + chunk, xw.shape[0])
            m = None if mask is None else mask[torch.arange(i, j, device=xw.device) % nw]
            with torch.enable_grad():
                x, t = xw[i:j].detach().requires_grad_(True), table.detach().requires_grad_(True)
                gx, gt = torch.autograd.grad(_attention_core(x, t, rel, m, heads, fp16_rounding), (x, t), dout[i:j])
            dx[i:j] = gx
            dt += gt
        return dx, dt, None, None, None, None, None


def window_attention_core(qkv, qkv_bias, table, heads, window, shift, fp16_rounding=False, chunk=64):
    """qkv [B,D,H,W,3C] -> attention output [B,D,H,W,C]: SwinTransformerBlock.forward_part1 between the qkv and proj
    Linears (swin_unetr.py:554-606), i.e. the operator of the project's window-attention kernels, differentiable in qkv,
    qkv_bias ([3C] or None) and table ([T, heads]).
      * The reference pads after norm1 and before the qkv Linear, so a padding token's q/k/v is the qkv bias.  Written
        as pad(qkv - b) + b, autograd sends exactly the padding region's gradient to b.
      * fp16_rounding: round where the reference's autocast rounds: the bias (an fp16 Linear on a zero input returns
        fp16(b)), q * scale, and the probabilities before `@ v`.  The rounding has an identity gradient.
      * The window is clamped (and its shift dropped) on axes not larger than it; the relative-position index is the
        nominal window's, sliced [:n, :n] (swin_unetr.py:474)."""
    B, D, H, W, C3 = qkv.shape
    ws, ss = get_window_size((D, H, W), window, shift)
    b = torch.zeros(C3, dtype=qkv.dtype, device=qkv.device) if qkv_bias is None else qkv_bias.to(qkv.dtype)
    if fp16_rounding:
        b = _round16(b)
    pads = [(ws[i] - s % ws[i]) % ws[i] for i, s in enumerate((D, H, W))]
    x = F.pad(qkv - b, (0, 0, 0, pads[2], 0, pads[1], 0, pads[0])) + b
    dp, hp, wp = x.shape[1:4]
    shifted = any(s > 0 for s in ss)
    if shifted:
        x = torch.roll(x, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
    n = ws[0] * ws[1] * ws[2]
    rel = relative_position_index(window)[:n, :n].to(qkv.device)
    mask = compute_mask((dp, hp, wp), ws, ss).to(qkv.device, qkv.dtype) if shifted else None
    out = _ChunkedCore.apply(window_partition(x, ws), table.to(qkv.dtype), rel, mask, heads, fp16_rounding, chunk)
    x = window_reverse(out, ws, [B, dp, hp, wp])
    if shifted:
        x = torch.roll(x, shifts=ss, dims=(1, 2, 3))
    return x[:, :D, :H, :W, :]


def patch_merging(x, norm_w, norm_b, red_w):
    """The v0.9 `PatchMerging` the reference instantiates (downsample='merging'), INCLUDING its quirk: slices x5 and x6
    repeat the offsets of x2 and x3, so the (0,1,1) and (1,1,0) sub-lattices are never read — swin_unetr.py:717-731."""
    b, d, h, w, c = x.shape
    if (h % 2 == 1) or (w % 2 == 1) or (d % 2 == 1):
        x = F.pad(x, (0, 0, 0, w % 2, 0, h % 2, 0, d % 2))
    offs = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 0), (0, 0, 1), (1, 1, 1)]
    x = torch.cat([x[:, i::2, j::2, k::2, :] for i, j, k in offs], -1)
    x = F.layer_norm(x, (8 * c,), norm_w, norm_b)
    return F.linear(x, red_w)


def patch_merging_v2(x, norm_w, norm_b, red_w):
    """`PatchMergingV2` (itertools.product order) — swin_unetr.py:684-704; not used by the default constructor."""
    b, d, h, w, c = x.shape
    if (h % 2 == 1) or (w % 2 == 1) or (d % 2 == 1):
        x = F.pad(x, (0, 0, 0, w % 2, 0, h % 2, 0, d % 2))
    x = torch.cat([x[:, i::2, j::2, k::2, :] for i, j, k in itertools.product(range(2), range(2), range(2))], -1)
    x = F.layer_norm(x, (8 * c,), norm_w, norm_b)
    return F.linear(x, red_w)
