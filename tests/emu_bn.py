"""CPU emulation of the per-channel convolution and BatchNorm C-ABI ops (TEST INFRASTRUCTURE).

Installs tests/emu_ops.py (the shared conv / pool / upsample / loss emulation) and additionally patches the launch
wrappers of b200seg.batchnorm, so the 2D UNet's host orchestration (autograd algebra, running-statistic updates,
holder lookup) runs without a GPU.  Every op computes in fp64 and hands tensors of the working dtype to the next one,
as the kernels do.  The product never imports this file."""
import torch
import torch.nn.functional as F

import emu_ops


def _nc(t, C):
    return t[..., :C].permute(0, 4, 1, 2, 3)


def _nd(t):
    return t.permute(0, 2, 3, 4, 1).contiguous()


def _per_c(v):
    return v[None, :, None, None, None]


def _act(h, act):
    return F.relu(h) if act == 1 else h


def _mask(z, act):
    return (z > 0).to(z.dtype) if act == 1 else torch.ones_like(z)


def _z(x, table):
    return x * _per_c(table[:, 0].double()) + _per_c(table[:, 1].double())


def install(monkeypatch):
    ops = emu_ops.install(monkeypatch)
    from b200seg import batchnorm as bn
    from b200seg import unet2d

    def conv_pc_fwd(x, Cin, affine, act, wp, Cout, ksize, bias=None, residual=None, want_stats=True):
        taps = ksize[0] * ksize[1] * ksize[2]
        w = wp[0].view(taps, Cout, Cin).permute(1, 2, 0).reshape(Cout, Cin, *ksize)
        a = _nc(x, Cin).double()
        if affine is not None:
            a = _z(a, affine)
        a = _act(a, act).to(x.dtype)
        y = F.conv3d(a.double(), w.double(), padding=[k // 2 for k in ksize])
        if bias is not None:
            y = y + _per_c(bias.double())
        y = y.to(x.dtype).double()
        if residual is not None:
            y = y + _nc(residual, Cout).double()
        y = y.to(x.dtype)
        st = emu_ops._stats(y) if want_stats else None
        return _nd(y), st

    def conv_pc_wgrad(x, Cin, affine, act, dy, Cout, ksize, want_bias=False):
        a = _nc(x, Cin).double()
        if affine is not None:
            a = _z(a, affine)
        a = _act(a, act).to(x.dtype).double()
        g = _nc(dy, Cout).double()
        w = torch.zeros(Cout, Cin, *ksize, dtype=torch.float64, requires_grad=True)
        with torch.enable_grad():
            F.conv3d(a, w, padding=[k // 2 for k in ksize]).backward(g)
        db = g.sum((0, 2, 3, 4)).float() if want_bias else None
        return w.grad.float(), db

    def bn_fold(holder, sums, count):
        bn._check_holder(holder)
        if holder.training and count <= 1:
            raise ValueError("Expected more than 1 value per channel when training, got %d" % count)
        if holder.training:
            s = sums.sum(0)
            mean = s[:, 0] / count
            var = (s[:, 1] / count - mean * mean).clamp_min(0)
            m = holder.momentum
            holder.running_mean.copy_(((1 - m) * holder.running_mean.double() + m * mean).float())
            holder.running_var.copy_(((1 - m) * holder.running_var.double() + m * var * count / (count - 1)).float())
            holder.num_batches_tracked += 1
        else:
            mean, var = holder.running_mean.double(), holder.running_var.double()
        rstd = 1.0 / torch.sqrt(var + holder.eps)
        sc = holder.weight.detach().double() * rstd
        table = torch.stack([sc, holder.bias.detach().double() - mean * sc], 1).float()
        return table, torch.stack([mean, rstd], 1).float()

    def bn_apply(x, table, act):
        return _nd(_act(_z(_nc(x, x.shape[-1]).double(), table), act).to(x.dtype))

    def _dz(g, x, table, act):
        C = x.shape[-1]
        xs = _nc(x, C).double()
        gg = _nc(g, C).double()
        if table is not None:
            gg = gg * _mask(_z(xs, table), act)
        return gg, xs

    def bn_bwd_reduce(g, x, table, act, mean_rstd):
        dz, xs = _dz(g, x, table, act)
        xh = (xs - _per_c(mean_rstd[:, 0].double())) * _per_c(mean_rstd[:, 1].double())
        return torch.stack([dz.sum((0, 2, 3, 4)), (dz * xh).sum((0, 2, 3, 4))], 1)

    def bn_bwd_fold(sums, count, gamma, mean_rstd, training):
        s1, s2 = sums[:, 0], sums[:, 1]
        mean, rstd = mean_rstd[:, 0].double(), mean_rstd[:, 1].double()
        gr = gamma.detach().double() * rstd
        zero = torch.zeros_like(gr)
        coef = torch.stack([gr, -gr * rstd * s2 / count if training else zero, mean,
                            -gr * s1 / count if training else zero], 1)
        return s2.float(), s1.float(), coef

    def bn_bwd_apply(g, x, table, act, coef, add=None, out=None):
        dz, xs = _dz(g, x, table, act)
        dx = _per_c(coef[:, 0]) * dz + _per_c(coef[:, 1]) * (xs - _per_c(coef[:, 2])) + _per_c(coef[:, 3])
        if add is not None:
            dx = dx + _nc(add, x.shape[-1]).double()
        dx = _nd(dx.to(x.dtype))
        if out is None:
            return dx
        out.copy_(dx)
        return out

    for name, fn in dict(conv_pc_fwd=conv_pc_fwd, conv_pc_wgrad=conv_pc_wgrad, bn_fold=bn_fold, bn_apply=bn_apply,
                         bn_bwd_reduce=bn_bwd_reduce, bn_bwd_fold=bn_bwd_fold, bn_bwd_apply=bn_bwd_apply).items():
        monkeypatch.setattr(bn, name, fn)
    monkeypatch.setattr(unet2d, "MaxPoolFn", ops.MaxPoolFn)
    monkeypatch.setattr(unet2d, "UpCatFn", ops.UpCatFn)
    return ops
