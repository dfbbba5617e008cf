"""BatchNorm2d blocks of the 2D UNet / ResUNet (model/dim2/conv_layers.py:21-94) on libb200seg.so.

Activations are NDHWC buffers with D = 1, and every 2D convolution is a (1, kh, kw) convolution in the library's
per-channel mode (b200seg_conv3d_fwd_pc): BatchNorm + ReLU of a pre-activation block never exist as a tensor, the
consuming convolution's loader applies relu(x*s[c] + t[c]) from a [C][2] table.  That table is built by the forward fold
from the fp64 per-(sample, channel) sums the producing kernel already wrote, so a layer costs no extra pass over its
input.  The tables are per channel, so the tensor-core limits do not depend on the batch size.

The backward of a BatchNorm layer runs on the raw data gradient: one reduction pass (sum dz, sum dz*xhat per channel),
a fold to dgamma / dbeta and per-channel coefficients, and one elementwise pass that writes (or accumulates) dx.
"""
import torch

from . import _lib, ops
from ._lib import ACT_NONE, ACT_RELU, ALGO_AUTO, call
from .ops import _dt, _need_cuda, _p, _stream, new_stats


# ----------------------------------------------------------------------------- raw launches
def conv_pc_fwd(x, Cin, affine, act, wp, Cout, ksize, bias=None, residual=None, want_stats=True):
    """y = conv(act(x*s + t)) (+bias)(+residual) on a whole NDHWC tensor; affine is a [Cin,2] {s,t} table or None.
    wp is a (packed image, algo) pair from PackedWeights (packed with B=1).  Returns (y, y_sums [B,Cout,2] or None)."""
    _need_cuda(x)
    wimg, algo = wp
    B, D, H, W, x_ld = x.shape
    y = torch.empty(B, D, H, W, Cout, dtype=x.dtype, device=x.device)
    y_sums = new_stats(B, Cout, x.device) if want_stats else None
    call("b200seg_conv3d_fwd_pc", x.data_ptr(), x_ld, 0, _p(affine), act, wimg.data_ptr(), _p(bias),
         _p(residual), 0 if residual is None else residual.shape[-1], 0, y.data_ptr(), Cout, 0, _p(y_sums),
         B, D, H, W, Cin, Cout, ksize[0], ksize[1], ksize[2], _dt(x), algo, _stream())
    return y, y_sums


def conv_pc_wgrad(x, Cin, affine, act, dy, Cout, ksize, want_bias=False, algo=ALGO_AUTO):
    """dW (and db) of y = conv(act(x*s + t)) (+bias), in the parameter layout [Cout, Cin, kd, kh, kw]."""
    B, D, H, W, x_ld = x.shape
    dw = torch.zeros(Cout, Cin, *ksize, dtype=torch.float32, device=x.device)
    db = torch.zeros(Cout, dtype=torch.float32, device=x.device) if want_bias else None
    transformed = 1 if (affine is not None or act) else 0
    ws_bytes = _lib.load().b200seg_conv3d_wgrad_pc_workspace(x_ld, 0, transformed, dy.shape[-1], 0, 1 if want_bias else 0,
                                                             B, D, H, W, Cin, Cout, ksize[0], ksize[1], ksize[2], _dt(x),
                                                             algo)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
    call("b200seg_conv3d_wgrad_pc", x.data_ptr(), x_ld, 0, _p(affine), act, dy.data_ptr(), dy.shape[-1], 0,
         dw.data_ptr(), _p(db), B, D, H, W, Cin, Cout, ksize[0], ksize[1], ksize[2], _dt(x), algo, _p(ws), ws_bytes,
         _stream())
    return dw, db


def _check_holder(bn):
    if bn.momentum is None or not bn.affine or not bn.track_running_stats:
        raise ValueError("the H100 BatchNorm needs momentum set, affine=True and track_running_stats=True "
                         "(the nn.BatchNorm2d defaults of model/dim2/conv_layers.py)")


def bn_fold(bn, sums, count):
    """Forward fold of the BatchNorm holder `bn` (nn.BatchNorm2d) from fp64 sums [nb, C, 2] over `count` values per
    channel: in training, batch statistics (and the running buffers updated in place); in eval, the running statistics.
    Returns (table [C,2] {s,t}, mean_rstd [C,2])."""
    _check_holder(bn)
    training = bn.training
    C = bn.num_features
    if training and count <= 1:
        raise ValueError("Expected more than 1 value per channel when training, got %d" % count)
    dev = bn.weight.device
    table = torch.empty(C, 2, dtype=torch.float32, device=dev)
    mean_rstd = torch.empty(C, 2, dtype=torch.float32, device=dev)
    call("b200seg_batchnorm_fwd_fold", _p(sums), 0 if sums is None else sums.shape[0], C, float(count),
         bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
         bn.num_batches_tracked.data_ptr(), float(bn.momentum), float(bn.eps), 1 if training else 0,
         table.data_ptr(), mean_rstd.data_ptr(), _stream())
    return table, mean_rstd


def bn_apply(x, table, act):
    """y = act(x*s + t) materialised (post-activation SingleConv)."""
    B, D, H, W, C = x.shape
    y = torch.empty_like(x)
    call("b200seg_batchnorm_apply", x.data_ptr(), _dt(x), C, 0, table.data_ptr(), act, y.data_ptr(), C, 0,
         B * D * H * W, C, _stream())
    return y


def bn_bwd_reduce(g, x, table, act, mean_rstd):
    """{sum dz, sum dz*xhat} per channel, fp64 [C,2]; dz = g * act'(x*s + t)."""
    B, D, H, W, C = x.shape
    sums = ops.zeros_scratch((C, 2), torch.float64, x.device)
    call("b200seg_batchnorm_bwd_reduce", g.data_ptr(), g.shape[-1], 0, x.data_ptr(), C, 0, _dt(x), _p(table), act,
         mean_rstd.data_ptr(), B * D * H * W, C, sums.data_ptr(), _stream())
    return sums


def bn_bwd_fold(sums, count, gamma, mean_rstd, training):
    """(dgamma, dbeta, coef [C,4]) from the backward sums."""
    C = gamma.shape[0]
    dg = torch.empty(C, dtype=torch.float32, device=gamma.device)
    db = torch.empty(C, dtype=torch.float32, device=gamma.device)
    coef = torch.empty(C, 4, dtype=torch.float32, device=gamma.device)
    call("b200seg_batchnorm_bwd_fold", sums.data_ptr(), float(count), gamma.data_ptr(), mean_rstd.data_ptr(),
         1 if training else 0, C, dg.data_ptr(), db.data_ptr(), coef.data_ptr(), _stream())
    return dg, db, coef


def bn_bwd_apply(g, x, table, act, coef, add=None, out=None):
    """dx = a*dz + b*(x - mean) + k (+ add), written to `out` (which may be `add`) or a new tensor."""
    B, D, H, W, C = x.shape
    out = torch.empty_like(x) if out is None else out
    call("b200seg_batchnorm_bwd_apply", g.data_ptr(), g.shape[-1], 0, x.data_ptr(), C, 0, _dt(x), _p(table), act,
         coef.data_ptr(), _p(add), C, 0, out.data_ptr(), C, 0, B * D * H * W, C, _stream())
    return out


# ----------------------------------------------------------------------------- one BatchNorm layer, both directions
def _count(x):
    return x.numel() // x.shape[-1]


class _Sync:
    """The process group a training nn.SyncBatchNorm holder reduces over (convert_sync_batchnorm, train_ddp.py:352,357),
    as torch.nn.SyncBatchNorm decides it: only in training and only with more than one rank."""

    def __init__(self, group):
        self.group = group

    @staticmethod
    def of(holder):
        dist = torch.distributed
        if not (isinstance(holder, torch.nn.SyncBatchNorm) and holder.training and dist.is_available()
                and dist.is_initialized()):
            return None
        group = holder.process_group if holder.process_group is not None else dist.group.WORLD
        return _Sync(group) if dist.get_world_size(group) > 1 else None

    def all_reduce(self, t):
        torch.distributed.all_reduce(t, group=self.group)
        return t


def fold(holder, sums, count):
    """Forward of one BatchNorm layer from the per-(sample, channel) sums [B, C, 2] of its input.  Under SyncBatchNorm
    the per-channel sums and the count are added over the holder's process group first, so the statistics, the
    running-variance unbiasing and the table are those of the global batch.  Returns the layer state the backward
    needs: (table, mean_rstd, count, sync)."""
    sync = _Sync.of(holder)
    if sync is not None:
        sums = sync.all_reduce(sums.sum(0, keepdim=True))
        n = sync.all_reduce(torch.tensor([float(count)], dtype=torch.float64, device=sums.device))
        count = int(n.item())
    table, mr = bn_fold(holder, sums, count)
    return table, mr, count, sync


def backward(g, x, layer, gamma, training, act=ACT_RELU, add=None, out=None):
    """dx (written to `out`, plus `add`), dgamma and dbeta of one BatchNorm + act layer whose input was x and whose
    output's gradient (through act) is g.  Under SyncBatchNorm dgamma / dbeta are the local ones (DDP averages them, as
    for torch.nn.SyncBatchNorm) and dx uses the backward sums added over the process group."""
    table, mr, count, sync = layer
    sums = bn_bwd_reduce(g, x, table, act, mr)
    dg, db, coef = bn_bwd_fold(sums, count, gamma, mr, training)
    if sync is not None:
        _, _, coef = bn_bwd_fold(sync.all_reduce(sums), count, gamma, mr, training)
    return bn_bwd_apply(g, x, table, act, coef, add=add, out=out), dg, db


# ----------------------------------------------------------------------------- autograd Functions


class BNSingleConvFn(torch.autograd.Function):
    """SingleConv (post-activation): y = relu(BN(conv(x))).  The raw conv output r and its per-(b,c) sums are kept;
    the BN + ReLU is materialised by one elementwise pass."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, bn, packs, ksize):
        Cout, Cin = w.shape[0], w.shape[1]
        w_fwd, w_bwd = packs
        r, r_sums = conv_pc_fwd(x, Cin, None, ACT_NONE, w_fwd, Cout, ksize)
        table, mr, count, sync = fold(bn, r_sums, _count(r))
        y = bn_apply(r, table, ACT_RELU)
        ctx.save_for_backward(x, r, table, mr, gamma, w_bwd[0])
        ctx.meta = (Cin, Cout, ksize, x.requires_grad, w_bwd[1], bn.training, count, sync)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, r, table, mr, gamma, w_bwd = ctx.saved_tensors
        Cin, Cout, ksize, need_dx, algo_b, training, count, sync = ctx.meta
        dy = dy.contiguous()
        dr, dg, db = backward(dy, r, (table, mr, count, sync), gamma, training)
        dw, _ = conv_pc_wgrad(x, Cin, None, ACT_NONE, dr, Cout, ksize)
        dx = None
        if need_dx:
            dx, _ = conv_pc_fwd(dr, Cout, None, ACT_NONE, (w_bwd, algo_b), Cin, ksize, want_stats=False)
        return dx, dw, dg, db, None, None, None


class BNBasicBlockFn(torch.autograd.Function):
    """Pre-activation residual block: out = conv2(relu(bn2(conv1(relu(bn1(x)))))) + shortcut(x), with
    shortcut = identity or conv_s(relu(bn_s(x))).  bn1 and bn_s share the batch statistics of x but not gamma / beta,
    so conv1 and the shortcut are two launches on the same input.  x_sums are the per-(b,c) sums of x."""

    @staticmethod
    def forward(ctx, x, x_sums, w1, g1, b1, w2, g2, b2, ws, gs, bs, bns, packs, ksize):
        bn1, bn2, bn_s = bns
        Cout, Cin = w1.shape[0], w1.shape[1]
        n = _count(x)
        (w1_fwd, w1_bwd), (w2_fwd, w2_bwd), pk_s = packs
        l1 = fold(bn1, x_sums, n)
        t, t_sums = conv_pc_fwd(x, Cin, l1[0], ACT_RELU, w1_fwd, Cout, ksize)
        has_sc = ws is not None
        if has_sc:
            ls = fold(bn_s, x_sums, n)
            res, _ = conv_pc_fwd(x, Cin, ls[0], ACT_RELU, pk_s[0], Cout, ksize, want_stats=False)
        else:
            ls = None
            res = x
        l2 = fold(bn2, t_sums, n)
        out, out_sums = conv_pc_fwd(t, Cout, l2[0], ACT_RELU, w2_fwd, Cout, ksize, residual=res)
        saved = [x, t, l1[0], l1[1], l2[0], l2[1], g1, g2, w1_bwd[0], w2_bwd[0]]
        if has_sc:
            saved += [ls[0], ls[1], gs, pk_s[1][0]]
        ctx.save_for_backward(*saved)
        # per layer: (count, sync) of its fold and its holder's training flag
        ctx.meta = (Cin, Cout, ksize, has_sc, w1_bwd[1], w2_bwd[1], pk_s[1][1] if has_sc else None,
                    (l1[2:], bn1.training), (l2[2:], bn2.training), (ls[2:], bn_s.training) if has_sc else None)
        ctx.mark_non_differentiable(out_sums)
        return out, out_sums

    @staticmethod
    def backward(ctx, d_out, _):
        Cin, Cout, ksize, has_sc, algo1, algo2, algo_s, m1, m2, ms = ctx.meta
        saved = ctx.saved_tensors
        x, t, tab1, mr1, tab2, mr2, g1, g2, w1_bwd, w2_bwd = saved[:10]
        d_out = d_out.contiguous()
        # ---- conv2 on relu(bn2(t))
        dw2, _ = conv_pc_wgrad(t, Cout, tab2, ACT_RELU, d_out, Cout, ksize)
        gt, _ = conv_pc_fwd(d_out, Cout, None, ACT_NONE, (w2_bwd, algo2), Cout, ksize, want_stats=False)
        dt, dg2, db2 = backward(gt, t, (tab2, mr2) + m2[0], g2, m2[1])
        del gt
        # ---- conv1 on relu(bn1(x))
        dw1, _ = conv_pc_wgrad(x, Cin, tab1, ACT_RELU, dt, Cout, ksize)
        gx, _ = conv_pc_fwd(dt, Cout, None, ACT_NONE, (w1_bwd, algo1), Cin, ksize, want_stats=False)
        if has_sc:
            tab_s, mr_s, gs, ws_bwd = saved[10:]
            dx, dg1, db1 = backward(gx, x, (tab1, mr1) + m1[0], g1, m1[1])
            dws, _ = conv_pc_wgrad(x, Cin, tab_s, ACT_RELU, d_out, Cout, ksize)
            gxs, _ = conv_pc_fwd(d_out, Cout, None, ACT_NONE, (ws_bwd, algo_s), Cin, ksize, want_stats=False)
            _, dgs, dbs = backward(gxs, x, (tab_s, mr_s) + ms[0], gs, ms[1], add=dx, out=dx)
        else:
            dx, dg1, db1 = backward(gx, x, (tab1, mr1) + m1[0], g1, m1[1], add=d_out)
            dws = dgs = dbs = None
        return dx, None, dw1, dg1, db1, dw2, dg2, db2, dws, dgs, dbs, None, None, None


class PointwiseConvFn(torch.autograd.Function):
    """1x1 convolution with bias on a raw NDHWC tensor (up_block.conv_ch and outc of model/dim2/unet*.py)."""

    @staticmethod
    def forward(ctx, x, w, bias, packs):
        w_fwd, w_bwd = packs
        Cout, Cin = w.shape[0], w.shape[1]
        y, _ = conv_pc_fwd(x, Cin, None, ACT_NONE, w_fwd, Cout, (1, 1, 1), bias=bias, want_stats=False)
        ctx.save_for_backward(x, w_bwd[0])
        ctx.meta = (Cin, Cout, w_bwd[1])
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w_bwd = ctx.saved_tensors
        Cin, Cout, algo_b = ctx.meta
        dy = dy.contiguous()
        dw, db = conv_pc_wgrad(x, Cin, None, ACT_NONE, dy, Cout, (1, 1, 1), want_bias=True)
        dx, _ = conv_pc_fwd(dy, Cout, None, ACT_NONE, (w_bwd, algo_b), Cin, (1, 1, 1), want_stats=False)
        return dx, dw, db, None
