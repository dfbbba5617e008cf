"""Differentiable MedFormer operators over the C-ABI kernels (channels-last tensors, IN sums travel beside them).

Every Function here launches only libb200seg kernels; the pieces they mirror are cited per class.  Convention
shared with ops.py: a feature is a pair (x [B,D,H,W,C], stats double[B,C,2] or None); InstanceNorm (+ReLU) is never
materialised — consumers apply it in their loaders from the producer's sums, and differentiate through it in
their own backward (in_bwd_reduce / in_bwd_apply).
"""
import torch

from . import _lib
from ._lib import ACT_NONE, call
from .ops import (_dt, _need_cuda, _stream, conv3d_fwd, conv3d_wgrad, copy_channels, dw_weight, dwconv3d, dwconv3d_wgrad,
                  in_bwd_apply, in_bwd_reduce, instnorm_stats, zeros_scratch)


class ConvFn(torch.autograd.Function):
    """y = conv(act(IN(x))) (+bias) (+residual), `ConvNormAct(preact=True)` conv_layers.py:46-53 with any of
    norm/act switched off; several weights sharing the input run as one GEMM (outputs concatenated).  `co_pad`
    zero output channels are appended by the packer.  Returns (y, IN sums of y or None when the consumer does not
    normalise y: the statistics butterfly is a large part of the conv epilogue)."""

    @staticmethod
    def forward(ctx, x, x_stats, residual, bias, packs, ksize, act, co_pad, eps, want_stats, *weights):
        _need_cuda(x)
        Cin = weights[0].shape[1]
        couts = [w.shape[0] for w in weights]
        Cout = sum(couts) + co_pad
        w_fwd, w_bwd = packs
        if bias is not None and co_pad:
            bias_k = torch.zeros(Cout, dtype=torch.float32, device=x.device)
            bias_k[:Cout - co_pad] = bias.detach().float()
        else:
            bias_k = None if bias is None else bias.detach().float().contiguous()
        y, y_stats = conv3d_fwd(x, 0, Cin, x_stats, act, w_fwd, Cout, ksize, bias=bias_k, residual=residual, eps=eps,
                                want_stats=want_stats)
        ctx.save_for_backward(x, x_stats, w_bwd[0])
        ctx.meta = (Cin, Cout, couts, tuple(ksize), act, w_bwd[1], bias is not None, residual is not None,
                    ctx.needs_input_grad[0], eps)
        if y_stats is not None:
            ctx.mark_non_differentiable(y_stats)
        return y, y_stats

    @staticmethod
    def backward(ctx, dy, _):
        x, x_stats, w_bwd = ctx.saved_tensors
        Cin, Cout, couts, ksize, act, algo_b, has_bias, has_res, need_dx, eps = ctx.meta
        dy = dy.contiguous()
        dw, db = conv3d_wgrad(x, 0, Cin, x_stats, act, dy, 0, Cout, ksize, want_bias=has_bias, eps=eps)
        dws, off = [], 0
        for c in couts:
            dws.append(dw[off:off + c])
            off += c
        dx = None
        if need_dx:
            if x_stats is not None:
                g, bst = conv3d_fwd(dy, 0, Cout, None, ACT_NONE, (w_bwd, algo_b), Cin, ksize,
                                    dgrad_of=(x, 0, x_stats, act), eps=eps)
                dx = in_bwd_apply(g, x, 0, Cin, x_stats, bst, eps=eps)
            else:
                dx, _ = conv3d_fwd(dy, 0, Cout, None, ACT_NONE, (w_bwd, algo_b), Cin, ksize, want_stats=False)
        if has_bias:
            db = db[:off]
        return (dx, None, dy if has_res else None, db if has_bias else None, None, None, None, None, None, None, *dws)


class DwConvFn(torch.autograd.Function):
    """y = depthwise_conv(act(IN(x))): DepthwiseSeparableConv.depthwise conv_layers.py:135-143 on a normalised
    input (norm1 medformer_utils.py:126, PatchMerging.norm :173) and MBConv.depthwise (ConvNormAct preact with
    groups == channels, conv_layers.py:208)."""

    @staticmethod
    def forward(ctx, x, x_stats, weight, act, eps, want_stats=True):
        ks = tuple(weight.shape[2:])
        wt = dw_weight(weight)              # the [C,1,kd,kh,kw] parameter itself: no per-call transposed copy
        x = x.contiguous()
        y, y_stats = dwconv3d(x, wt, ks, x_stats=x_stats, act=act, want_stats=want_stats, eps=eps, cmajor=True)
        ctx.save_for_backward(x, x_stats, wt)
        ctx.meta = (ks, act, weight.dtype, eps)
        if y_stats is not None:
            ctx.mark_non_differentiable(y_stats)
        return y, y_stats

    @staticmethod
    def backward(ctx, dy, _):
        x, x_stats, wt = ctx.saved_tensors
        ks, act, wdtype, eps = ctx.meta
        dy = dy.contiguous()
        C = x.shape[-1]
        dw = dwconv3d_wgrad(x, dy, ks, x_stats=x_stats, act=act, eps=eps, cmajor=True)
        g, _ = dwconv3d(dy, wt, ks, flip=True, cmajor=True)
        if x_stats is not None:
            g2, bst = in_bwd_reduce(g, x, C, x_stats, act, eps=eps)
            dx = in_bwd_apply(g2, x, 0, C, x_stats, bst, eps=eps)
        else:
            dx = g
        return dx, None, dw.to(wdtype), None, None, None


class SpaceToDepthFn(torch.autograd.Function):
    """PatchMerging's strided-slice gather + cat, medformer_utils.py:165-171, with the IN sums of the result."""

    @staticmethod
    def forward(ctx, x, scale):
        _need_cuda(x)
        x = x.contiguous()
        B, D, H, W, C = x.shape
        sd, sh, sw = scale
        if D % sd or H % sh or W % sw:
            raise ValueError("PatchMerging needs extents divisible by the down scale (torch.cat would fail too)")
        Do, Ho, Wo = D // sd, H // sh, W // sw
        y = torch.empty(B, Do, Ho, Wo, C * sd * sh * sw, dtype=x.dtype, device=x.device)
        call("b200seg_space_to_depth", x.data_ptr(), y.data_ptr(), B, Do, Ho, Wo, C, sd, sh, sw, 0, _dt(x), _stream())
        st = instnorm_stats(y, 0, y.shape[-1])
        ctx.meta = (x.shape, scale)
        ctx.mark_non_differentiable(st)
        return y, st

    @staticmethod
    def backward(ctx, dy, _):
        (B, D, H, W, C), (sd, sh, sw) = ctx.meta
        dy = dy.contiguous()
        dx = torch.empty(B, D, H, W, C, dtype=dy.dtype, device=dy.device)
        call("b200seg_space_to_depth", dx.data_ptr(), dy.data_ptr(), B, D // sd, H // sh, W // sw, C, sd, sh, sw, 1,
             _dt(dy), _stream())
        return dx, None


class MapGenFn(torch.autograd.Function):
    """semantic_map = einsum('bij,bkj->bik', feat, softmax_j(weight_map)), medformer_utils.py:221-226, from the
    fused projection output fw = [base_proj(x) | semantic_proj(x) | zero pad] (channels C, K, pad)."""

    @staticmethod
    def forward(ctx, fw, C, K, map_size):
        _need_cuda(fw)
        fw = fw.contiguous()
        B = fw.shape[0]
        ld = fw.shape[-1]
        N = fw.numel() // (B * ld)
        smap = torch.empty(B, *map_size, C, dtype=fw.dtype, device=fw.device)
        colstat = torch.empty(B, K, 2, dtype=torch.float32, device=fw.device)
        ws = torch.empty(_lib.load().b200seg_mapgen_workspace(B, N, K, C), dtype=torch.uint8, device=fw.device)
        call("b200seg_mapgen_fwd", fw.data_ptr(), ld, 0, fw.data_ptr(), ld, C, smap.data_ptr(), colstat.data_ptr(),
             ws.data_ptr(), B, N, K, C, _dt(fw), _stream())
        ctx.save_for_backward(fw, smap, colstat)
        ctx.meta = (C, K)
        return smap

    @staticmethod
    def backward(ctx, dmap):
        fw, smap, colstat = ctx.saved_tensors
        C, K = ctx.meta
        dmap = dmap.contiguous()
        B, ld = fw.shape[0], fw.shape[-1]
        N = fw.numel() // (B * ld)
        dfw = torch.empty_like(fw)
        call("b200seg_mapgen_bwd", fw.data_ptr(), ld, 0, fw.data_ptr(), ld, C, smap.data_ptr(), colstat.data_ptr(),
             dmap.data_ptr(), dfw.data_ptr(), ld, 0, dfw.data_ptr(), ld, C, ld - C, B, N, K, C, _dt(fw), _stream())
        return dfw, None, None, None


class SEScaleFn(torch.autograd.Function):
    """SEBlock conv_layers.py:159-174: y = x * sigmoid(W2 relu(W1 avgpool(x) + b1) + b2).  The pooled means come
    from x's IN sums; the sums of y follow analytically (gate and gate^2)."""

    @staticmethod
    def forward(ctx, x, x_stats, w1, b1, w2, b2):
        _need_cuda(x)
        x = x.contiguous()
        B, D, H, W, C = x.shape
        V = D * H * W
        R = w1.shape[0]
        f = [t.detach().float().contiguous() for t in (w1, b1, w2, b2)]
        gate = torch.empty(B, C, dtype=torch.float32, device=x.device)
        hidden = torch.empty(B, R, dtype=torch.float32, device=x.device)
        mean = torch.empty(B, C, dtype=torch.float32, device=x.device)
        call("b200seg_se_gate_fwd", x_stats.data_ptr(), V, f[0].data_ptr(), f[1].data_ptr(), f[2].data_ptr(),
             f[3].data_ptr(), gate.data_ptr(), hidden.data_ptr(), mean.data_ptr(), B, C, R, _stream())
        y = torch.empty_like(x)
        call("b200seg_channel_scale_fwd", x.data_ptr(), gate.data_ptr(), y.data_ptr(), B, V, C, _dt(x), _stream())
        y_stats = instnorm_stats(y, 0, C)
        ctx.save_for_backward(x, gate, hidden, mean, f[0], f[2])
        ctx.meta = (w1.shape, w2.shape, w1.dtype)
        ctx.mark_non_differentiable(y_stats)
        return y, y_stats

    @staticmethod
    def backward(ctx, dy, _):
        x, gate, hidden, mean, w1, w2 = ctx.saved_tensors
        s1, s2, wdtype = ctx.meta
        dy = dy.contiguous()
        B, D, H, W, C = x.shape
        V = D * H * W
        R = s1[0]
        dev = x.device
        dgate = zeros_scratch((B, C), torch.float32, dev)
        ws = torch.empty(_lib.load().b200seg_channel_scale_bwd_workspace(B, V, C), dtype=torch.uint8, device=dev)
        call("b200seg_channel_scale_bwd_reduce", dy.data_ptr(), x.data_ptr(), dgate.data_ptr(), ws.data_ptr(), B, V, C,
             _dt(x), _stream())
        dw1 = torch.zeros(R, C, dtype=torch.float32, device=dev)
        db1 = torch.zeros(R, dtype=torch.float32, device=dev)
        dw2 = torch.zeros(C, R, dtype=torch.float32, device=dev)
        db2 = torch.zeros(C, dtype=torch.float32, device=dev)
        dmean = torch.empty(B, C, dtype=torch.float32, device=dev)
        call("b200seg_se_gate_bwd", dgate.data_ptr(), gate.data_ptr(), hidden.data_ptr(), mean.data_ptr(),
             w1.data_ptr(), w2.data_ptr(), dw1.data_ptr(), db1.data_ptr(), dw2.data_ptr(), db2.data_ptr(),
             dmean.data_ptr(), B, C, R, _stream())
        dx = torch.empty_like(x)
        call("b200seg_channel_scale_bwd_apply", dy.data_ptr(), gate.data_ptr(), dmean.data_ptr(), dx.data_ptr(),
             B, V, C, _dt(x), _stream())
        return dx, None, dw1.reshape(s1).to(wdtype), db1.to(wdtype), dw2.reshape(s2).to(wdtype), db2.to(wdtype)


class UpsampleFn(torch.autograd.Function):
    """F.interpolate(x, size, mode='trilinear', align_corners=True) for the auxiliary head, medformer.py:86."""

    @staticmethod
    def forward(ctx, x, size):
        _need_cuda(x)
        x = x.contiguous()
        B, Di, Hi, Wi, C = x.shape
        Do, Ho, Wo = size
        y = torch.empty(B, Do, Ho, Wo, C, dtype=x.dtype, device=x.device)
        call("b200seg_upsample_trilinear_fwd", x.data_ptr(), C, 0, y.data_ptr(), C, 0, None,
             B, Di, Hi, Wi, Do, Ho, Wo, C, _dt(x), _stream())
        ctx.meta = (x.shape, size)
        return y

    @staticmethod
    def backward(ctx, dy):
        (B, Di, Hi, Wi, C), (Do, Ho, Wo) = ctx.meta
        dy = dy.contiguous()
        dx = torch.empty(B, Di, Hi, Wi, C, dtype=dy.dtype, device=dy.device)
        call("b200seg_upsample_trilinear_bwd", dy.data_ptr(), C, 0, dx.data_ptr(), C, 0, 0,
             B, Di, Hi, Wi, Do, Ho, Wo, C, _dt(dy), _stream())
        return dx, None


class LayerNormFn(torch.autograd.Function):
    """nn.LayerNorm(dim) of PreNorm, trans_layers.py:36-41 (eps 1e-5), over tokens [B,L,C]."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        _need_cuda(x)
        x = x.contiguous()
        C = x.shape[-1]
        R = x.numel() // C
        g, b = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
        y = torch.empty_like(x)
        mr = torch.empty(R, 2, dtype=torch.float32, device=x.device)
        call("b200seg_layernorm_fwd", x.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), mr.data_ptr(), R, C,
             eps, _dt(x), _stream())
        ctx.save_for_backward(x, g, mr)
        ctx.wdtype = gamma.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g, mr = ctx.saved_tensors
        dy = dy.contiguous()
        C = x.shape[-1]
        R = x.numel() // C
        dx = torch.empty_like(x)
        dg = torch.zeros(C, dtype=torch.float32, device=x.device)
        db = torch.zeros(C, dtype=torch.float32, device=x.device)
        call("b200seg_layernorm_bwd", dy.data_ptr(), x.data_ptr(), g.data_ptr(), mr.data_ptr(), dx.data_ptr(),
             dg.data_ptr(), db.data_ptr(), R, C, _dt(x), _stream())
        return dx, dg.to(ctx.wdtype), db.to(ctx.wdtype), None


class GeluFn(torch.autograd.Function):
    """nn.GELU() (exact) of Mlp, trans_layers.py:22,28."""

    @staticmethod
    def forward(ctx, x):
        _need_cuda(x)
        x = x.contiguous()
        y = torch.empty_like(x)
        call("b200seg_gelu", x.data_ptr(), None, y.data_ptr(), x.numel(), _dt(x), _stream())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        call("b200seg_gelu", x.data_ptr(), dy.data_ptr(), dx.data_ptr(), x.numel(), _dt(x), _stream())
        return dx


class MHSAFn(torch.autograd.Function):
    """softmax(q k^T * scale) v per head over the fused map tokens, trans_layers.py:84-93.  qkv [B,L,3*inner]."""

    @staticmethod
    def forward(ctx, qkv, heads, dim_head):
        _need_cuda(qkv)
        qkv = qkv.contiguous()
        B, L = qkv.shape[0], qkv.shape[1]
        out = torch.empty(B, L, heads * dim_head, dtype=qkv.dtype, device=qkv.device)
        call("b200seg_mhsa", qkv.data_ptr(), None, out.data_ptr(), None, B, L, heads, dim_head,
             float(dim_head) ** -0.5, _dt(qkv), _stream())
        ctx.save_for_backward(qkv)
        ctx.hd = (heads, dim_head)
        return out

    @staticmethod
    def backward(ctx, dout):
        (qkv,) = ctx.saved_tensors
        heads, dim_head = ctx.hd
        dout = dout.contiguous()
        B, L = qkv.shape[0], qkv.shape[1]
        dqkv = torch.empty_like(qkv)
        call("b200seg_mhsa", qkv.data_ptr(), dout.data_ptr(), None, dqkv.data_ptr(), B, L, heads, dim_head,
             float(dim_head) ** -0.5, _dt(qkv), _stream())
        return dqkv, None, None


class AddFn(torch.autograd.Function):
    """a + b for two same-shape channels-last tensors (the map residuals, medformer_utils.py:136; token
    residuals trans_layers.py:113-114 when not already fused into a conv epilogue)."""

    @staticmethod
    def forward(ctx, a, b):
        out = a.contiguous().clone()
        copy_channels(b.contiguous(), 0, out, 0, out.shape[-1], accumulate=True)
        return out

    @staticmethod
    def backward(ctx, d):
        return d, d


class CatFn(torch.autograd.Function):
    """torch.cat([a, b], channel) for small channels-last tensors (map concat medformer_utils.py:395; token concat
    along L is a plain view in channels-last, see SemanticMapFusion)."""

    @staticmethod
    def forward(ctx, a, b):
        Ca, Cb = a.shape[-1], b.shape[-1]
        out = torch.empty(*a.shape[:-1], Ca + Cb, dtype=a.dtype, device=a.device)
        copy_channels(a.contiguous(), 0, out, 0, Ca)
        copy_channels(b.contiguous(), 0, out, Ca, Cb)
        ctx.split = (Ca, Cb)
        return out

    @staticmethod
    def backward(ctx, d):
        Ca, Cb = ctx.split
        d = d.contiguous()
        da = torch.empty(*d.shape[:-1], Ca, dtype=d.dtype, device=d.device)
        db = torch.empty(*d.shape[:-1], Cb, dtype=d.dtype, device=d.device)
        copy_channels(d, 0, da, 0, Ca)
        copy_channels(d, Ca, db, 0, Cb)
        return da, db
