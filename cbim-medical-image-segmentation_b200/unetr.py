"""UNETR whose every op runs in libb200seg.so — drop-in for the reference's ``model/dim3/unetr.py`` (the class
``get_model`` builds at model/utils.py): same constructor signature, same module tree, therefore the same
``state_dict`` keys / shapes / registration order — including the modules the reference takes from ``monai`` 1.1.0
(ViT, PatchEmbeddingBlock, TransformerBlock, SABlock, MLPBlock, UnetrBasicBlock, UnetrPrUpBlock, UnetrUpBlock,
UnetOutBlock), re-created here under their MONAI attribute names.  MONAI's source is not part of the reference, so
those blocks follow its published 1.1.0 semantics ("parity unpinned", as for SwinUNETR); the wiring the reference
file itself defines is pinned (oracle/make_golden_unetr.py).

Underneath: the ViT runs on the token matrix [B*L, hidden] viewed as a [1, 1, M/W, W, hidden] channels-last tensor,
so every Linear (patch embedding, qkv, out_proj, linear1/2) is a 1x1x1 tensor-core GEMM over 16x8 output tiles with
bias / residual in the epilogue; the position embedding is that GEMM's residual; attention is one global-attention
kernel between qkv and out_proj (csrc/attention.cu).  The token order is the NDHWC order of the 16^3 patch grid, so
``proj_feat`` is a free view; the decoder is SwinUNETR's MONAI blocks."""
import torch
import torch.nn as nn

from . import ops
from ._lib import ACT_NONE, call
from .medformer_ops import ConvFn
from .ops import PackedWeights, _dt, _need_cuda, _stream
from .swin_unetr import (IN_EPS, Convolution, DeriveWeightFn, DepthSpaceFn, MLPBlock, UnetOutBlock, UnetrBasicBlock,
                         UnetrUpBlock, _linear, _ln)

PATCH = 16
DIM_HEAD = 64          # the head size b200seg_attention implements (UNETR: 768 / 12)


def _flat(M):
    """[1, 1, M/W, W] token view of M tokens: W = 8 fills the GEMM's 16x8 output tiles whatever L is."""
    W = 8 if M % 8 == 0 else 1
    return (1, 1, M // W, W)


# ----------------------------------------------------------------------------- autograd Functions
class AttentionFn(torch.autograd.Function):
    """SABlock.forward between its two Linears: qkv (tokens of batch element b are rows b*L .. b*L+L-1 of the token
    matrix, channel which*inner + h*64 + d) -> softmax(q k^T / 8) v with channel h*64 + d."""

    @staticmethod
    def forward(ctx, qkv, B, heads):
        _need_cuda(qkv)
        qkv = qkv.contiguous()
        C3 = qkv.shape[-1]
        L = qkv.numel() // (B * C3)
        dh = C3 // (3 * heads)
        out = torch.empty(*qkv.shape[:-1], C3 // 3, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(B, heads, L, dtype=torch.float32, device=qkv.device)
        call("b200seg_attention_fwd", qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, L, heads, dh, _dt(qkv), _stream())
        ctx.save_for_backward(qkv, out, lse)
        ctx.meta = (B, L, heads, dh)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, lse = ctx.saved_tensors
        B, L, heads, dh = ctx.meta
        dout = dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse)
        call("b200seg_attention_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), delta.data_ptr(),
             dqkv.data_ptr(), B, L, heads, dh, _dt(qkv), _stream())
        return dqkv, None, None


class PatchifyFn(torch.autograd.Function):
    """PatchEmbeddingBlock's Rearrange 'b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)' on a channels-last volume:
    space-to-depth by 16 with channel ((p1*16 + p2)*16 + p3)*C + c; the (h w d) token order is the NDHWC grid order."""

    @staticmethod
    def forward(ctx, x):
        _need_cuda(x)
        x = x.contiguous()
        B, D, H, W, C = x.shape
        P = PATCH
        y = torch.empty(B, D // P, H // P, W // P, P ** 3 * C, dtype=x.dtype, device=x.device)
        call("b200seg_space_to_depth", x.data_ptr(), y.data_ptr(), B, D // P, H // P, W // P, C, P, P, P, 0, _dt(x), _stream())
        ctx.shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        B, D, H, W, C = ctx.shape
        P = PATCH
        dy = dy.contiguous()
        dx = torch.empty(B, D, H, W, C, dtype=dy.dtype, device=dy.device)
        call("b200seg_space_to_depth", dx.data_ptr(), dy.data_ptr(), B, D // P, H // P, W // P, C, P, P, P, 1, _dt(dy), _stream())
        return dx


class PosEmbedFn(torch.autograd.Function):
    """The [1, L, C] position table broadcast over the batch into a persistent [B, L, C] buffer (the patch GEMM's
    residual, stable address like DeriveWeightFn's).  Its gradient is the batch sum of the residual gradient,
    accumulated in batch order, so it is the same on every run."""

    @staticmethod
    def forward(ctx, table, buf, shape):
        B, L, C = buf.shape
        t = table.detach().float().contiguous().view(L, C)
        for b in range(B):
            ops.copy_channels(t, 0, buf[b], 0, C)
        ctx.meta = (tuple(buf.shape), table.dtype)
        return buf.view(shape)

    @staticmethod
    def backward(ctx, d):
        (B, L, C), tdtype = ctx.meta
        d = d.contiguous().view(B, L, C)
        g = torch.empty(L, C, dtype=torch.float32, device=d.device)
        for b in range(B):
            ops.copy_channels(d[b], 0, g, 0, C, accumulate=b > 0)
        return g.view(1, L, C).to(tdtype), None, None


def _up2(free, wt, x):
    """ConvTranspose3d(k2, s2, no bias) as UnetrUpBlock.forward runs it: permuted weight -> 1x1 GEMM -> depth-to-space."""
    ci, co = wt.shape[:2]
    if free["buf"] is None or free["buf"].device != x.device:
        free["buf"] = torch.empty(8 * co, ci, 1, 1, 1, dtype=torch.float32, device=x.device)
    w = DeriveWeightFn.apply(wt, (2, 3, 4, 1, 0), (8 * co, ci, 1, 1, 1), free["buf"])   # row q*Cout + co
    packs = free["pack"].get([w], x.dtype, x.shape[0], 0)
    y8, _ = ConvFn.apply(x, None, None, None, packs, (1, 1, 1), ACT_NONE, 0, IN_EPS, False, w)
    return DepthSpaceFn.apply(y8, False)


def _trunc_normal(t):
    """monai's trunc_normal_(mean 0, std 0.02, a -2, b 2): the same draws as torch's"""
    nn.init.trunc_normal_(t, mean=0.0, std=0.02, a=-2.0, b=2.0)


# ----------------------------------------------------------------------------- MONAI-named blocks
class _Rearrange(nn.Module):
    """Stateless stand-in for PatchEmbeddingBlock's einops Rearrange (index 0 of `patch_embeddings`)."""


class PatchEmbeddingBlock(nn.Module):
    """monai PatchEmbeddingBlock(pos_embed='perceptron', dropout 0): registration order patch_embeddings
    (Rearrange, Linear), position_embeddings, dropout; state_dict puts position_embeddings first."""

    def __init__(self, in_channels, img_size, patch_size, hidden_size, num_heads, pos_embed, dropout_rate=0.0, spatial_dims=3):
        super().__init__()
        self.n_patches = 1
        for m, p in zip(img_size, patch_size):
            self.n_patches *= m // p
        self.patch_dim = in_channels * patch_size[0] * patch_size[1] * patch_size[2]
        self.patch_embeddings = nn.Sequential(_Rearrange(), nn.Linear(self.patch_dim, hidden_size))
        self.position_embeddings = nn.Parameter(torch.zeros(1, self.n_patches, hidden_size))
        self.dropout = nn.Dropout(dropout_rate)
        _trunc_normal(self.position_embeddings)
        self.apply(self._init_weights)
        self._pack = PackedWeights()
        self._free = {"buf": None}

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            _trunc_normal(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, x):
        """x [B, D, H, W, Cin] -> tokens [1, 1, M/W, W, hidden] (x + position_embeddings)"""
        xs = PatchifyFn.apply(x)
        B, C = x.shape[0], self.position_embeddings.shape[-1]
        M = xs.numel() // xs.shape[-1]
        shape = _flat(M) + (C,)
        buf = self._free["buf"]
        if buf is None or buf.shape[0] != B or buf.dtype != x.dtype or buf.device != x.device:
            buf = self._free["buf"] = torch.empty(B, M // B, C, dtype=x.dtype, device=x.device)
        pos = PosEmbedFn.apply(self.position_embeddings, buf, shape)
        return _linear(self._pack, xs.view(*shape[:-1], xs.shape[-1]), self.patch_embeddings[1], residual=pos)


class SABlock(nn.Module):
    """monai SABlock(hidden, heads, dropout 0, qkv_bias False): out_proj, qkv, drop_output, drop_weights."""

    def __init__(self, hidden_size, num_heads, dropout_rate=0.0, qkv_bias=False):
        super().__init__()
        self.num_heads = num_heads
        self.out_proj = nn.Linear(hidden_size, hidden_size)
        self.qkv = nn.Linear(hidden_size, hidden_size * 3, bias=qkv_bias)
        self.drop_output = nn.Dropout(dropout_rate)
        self.drop_weights = nn.Dropout(dropout_rate)
        self.head_dim = hidden_size // num_heads
        self.scale = self.head_dim ** -0.5
        self._pq, self._po = PackedWeights(), PackedWeights()

    def forward(self, xn, shortcut, B):
        """xn = norm1(x) tokens; returns shortcut + out_proj(attention(qkv(xn)))."""
        att = AttentionFn.apply(_linear(self._pq, xn, self.qkv), B, self.num_heads)
        return _linear(self._po, att, self.out_proj, residual=shortcut)


class TransformerBlock(nn.Module):
    """monai TransformerBlock: mlp, norm1, attn, norm2;  x + attn(norm1(x)), then x + mlp(norm2(x))."""

    def __init__(self, hidden_size, mlp_dim, num_heads, dropout_rate=0.0, qkv_bias=False):
        super().__init__()
        self.mlp = MLPBlock(hidden_size, mlp_dim)
        self.norm1 = nn.LayerNorm(hidden_size)
        self.attn = SABlock(hidden_size, num_heads, dropout_rate, qkv_bias)
        self.norm2 = nn.LayerNorm(hidden_size)

    def forward(self, x, B):
        x = self.attn(_ln(x, self.norm1), x, B)
        return self.mlp(_ln(x, self.norm2), x)


class ViT(nn.Module):
    """monai ViT (classification=False): patch_embedding, blocks, norm.  forward returns (norm(last), per-block
    hidden states), all as [1, 1, M/W, W, hidden] token views."""

    def __init__(self, in_channels, img_size, patch_size, hidden_size=768, mlp_dim=3072, num_layers=12, num_heads=12,
                 pos_embed="perceptron", classification=False, dropout_rate=0.0, spatial_dims=3, qkv_bias=False):
        super().__init__()
        if classification:
            raise ValueError("the H100 path implements the ViT UNETR builds (classification=False)")
        self.classification = classification
        self.patch_embedding = PatchEmbeddingBlock(in_channels, img_size, patch_size, hidden_size, num_heads, pos_embed,
                                                   dropout_rate, spatial_dims)
        self.blocks = nn.ModuleList([TransformerBlock(hidden_size, mlp_dim, num_heads, dropout_rate, qkv_bias)
                                     for _ in range(num_layers)])
        self.norm = nn.LayerNorm(hidden_size)

    def forward(self, x):
        B = x.shape[0]
        t = self.patch_embedding(x)
        hidden_states_out = []
        for blk in self.blocks:
            t = blk(t, B)
            hidden_states_out.append(t)
        return _ln(t, self.norm), hidden_states_out


class UnetrPrUpBlock(nn.Module):
    """monai UnetrPrUpBlock(conv_block=False): transp_conv_init, then `num_layer` more bias-free k2s2 transposed convs."""

    def __init__(self, spatial_dims, in_channels, out_channels, num_layer, kernel_size, stride, upsample_kernel_size,
                 norm_name, conv_block=False, res_block=False):
        super().__init__()
        if spatial_dims != 3 or upsample_kernel_size != 2 or conv_block:
            raise ValueError("the H100 path implements the UnetrPrUpBlock configuration UNETR uses (3D, up 2, conv_block=False)")
        self.transp_conv_init = Convolution(in_channels, out_channels, 2, transposed=True)
        self.blocks = nn.ModuleList([Convolution(out_channels, out_channels, 2, transposed=True) for _ in range(num_layer)])
        # a dict keeps these holders out of the model's PackRegistry: they pack the derived weight buffer, which is
        # only refreshed inside forward (as in SwinUNETR's UnetrUpBlock)
        self._free = {"stages": [{"pack": PackedWeights(), "buf": None} for _ in range(num_layer + 1)]}

    def forward(self, x):
        for free, conv in zip(self._free["stages"], [self.transp_conv_init, *self.blocks]):
            x = _up2(free, conv.conv.weight, x)
        return x


# ----------------------------------------------------------------------------- the reference class
class UNETR(nn.Module):
    """model/dim3/unetr.py:22-237."""

    def __init__(self, in_channels, out_channels, img_size, feature_size=16, hidden_size=768, mlp_dim=3072, num_heads=12,
                 pos_embed="perceptron", norm_name="instance", conv_block=False, res_block=True, dropout_rate=0.0):
        super().__init__()
        if not (0 <= dropout_rate <= 1):
            raise AssertionError("dropout_rate should be between 0 and 1.")
        if hidden_size % num_heads != 0:
            raise AssertionError("hidden size should be divisible by num_heads.")
        if pos_embed not in ["conv", "perceptron"]:
            raise KeyError(f"Position embedding layer of type {pos_embed} is not supported.")
        if pos_embed != "perceptron":
            raise ValueError("the H100 path implements pos_embed='perceptron' only (the reference's get_model call)")
        if conv_block:
            raise ValueError("the H100 path implements conv_block=False only (the reference's default)")
        if dropout_rate:
            raise ValueError("dropout is not implemented by the H100 path (the reference trains UNETR with 0)")
        if hidden_size // num_heads != DIM_HEAD:
            raise ValueError("the H100 attention kernel implements head size %d, got hidden_size / num_heads = %d"
                             % (DIM_HEAD, hidden_size // num_heads))
        img_size = tuple(img_size) if isinstance(img_size, (list, tuple)) else (img_size,) * 3
        if len(img_size) != 3 or any(m % PATCH for m in img_size):
            raise ValueError("img_size should be 3D and divisible by the patch size %d, got %r" % (PATCH, img_size))
        self.num_layers = 12
        self.patch_size = (PATCH, PATCH, PATCH)
        self.img_size = img_size
        self.feat_size = tuple(m // PATCH for m in img_size)
        self.hidden_size = hidden_size
        self.classification = False
        self.vit = ViT(in_channels=in_channels, img_size=img_size, patch_size=self.patch_size, hidden_size=hidden_size,
                       mlp_dim=mlp_dim, num_layers=self.num_layers, num_heads=num_heads, pos_embed=pos_embed,
                       classification=self.classification, dropout_rate=dropout_rate)
        self.encoder1 = UnetrBasicBlock(spatial_dims=3, in_channels=in_channels, out_channels=feature_size, kernel_size=3,
                                        stride=1, norm_name=norm_name, res_block=res_block)
        pr = dict(spatial_dims=3, in_channels=hidden_size, kernel_size=3, stride=1, upsample_kernel_size=2,
                  norm_name=norm_name, conv_block=conv_block, res_block=res_block)
        self.encoder2 = UnetrPrUpBlock(out_channels=feature_size * 2, num_layer=2, **pr)
        self.encoder3 = UnetrPrUpBlock(out_channels=feature_size * 4, num_layer=1, **pr)
        self.encoder4 = UnetrPrUpBlock(out_channels=feature_size * 8, num_layer=0, **pr)
        up = dict(spatial_dims=3, kernel_size=3, upsample_kernel_size=2, norm_name=norm_name, res_block=res_block)
        self.decoder5 = UnetrUpBlock(in_channels=hidden_size, out_channels=feature_size * 8, **up)
        self.decoder4 = UnetrUpBlock(in_channels=feature_size * 8, out_channels=feature_size * 4, **up)
        self.decoder3 = UnetrUpBlock(in_channels=feature_size * 4, out_channels=feature_size * 2, **up)
        self.decoder2 = UnetrUpBlock(in_channels=feature_size * 2, out_channels=feature_size, **up)
        self.out = UnetOutBlock(spatial_dims=3, in_channels=feature_size, out_channels=out_channels)
        self._packs = ops.PackRegistry(self)

    def forward(self, x_in):
        if not x_in.is_cuda:
            raise ops._lib.B200SegError("b200seg.UNETR runs on an H100 only — there is no CPU fallback")
        if tuple(x_in.shape[2:]) != self.img_size:
            raise ValueError("UNETR was built for img_size %r, got an input of %r" % (self.img_size, tuple(x_in.shape[2:])))
        with ops.on_device(x_in):
            return self._forward(x_in)

    def _forward(self, x_in):
        dt = ops.compute_dtype()
        self._packs.refresh()
        x = x_in.permute(0, 2, 3, 4, 1).to(dt).contiguous()                # NDHWC working layout
        grid = (x.shape[0],) + self.feat_size + (self.hidden_size,)

        def proj_feat(t):                                                    # the token matrix IS the NDHWC patch grid
            return t.view(grid)
        last, hs = self.vit(x)
        enc1 = self.encoder1(x)
        enc2 = self.encoder2(proj_feat(hs[3]))
        enc3 = self.encoder3(proj_feat(hs[6]))
        enc4 = self.encoder4(proj_feat(hs[9]))
        dec3 = self.decoder5(proj_feat(last), enc4)
        dec2 = self.decoder4(dec3, enc3)
        dec1 = self.decoder3(dec2, enc2)
        out = self.decoder2(dec1, enc1)
        return self.out(out).permute(0, 4, 1, 2, 3)                         # logical NCDHW over the NDHWC buffer
