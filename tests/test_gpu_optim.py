"""GPU: the fused optimiser tail (SURVEY.md §8f.1) against the reference loop's own pieces step by step —
torch.optim.AdamW(eps=1e-5, weight_decay=0.05) (training/utils.py:8-14), torch.amp.GradScaler
(train_ddp.py:193-195) and update_ema_variables (training/utils.py:98-105) — including a step whose gradients
overflow (skipped by both, loss scale halved, EMA still updated).

Both kernels work on 8 192-element chunks, with float4 loads when a tensor's size is a multiple of 4 and scalar ones
otherwise.  The shape sets cover one-chunk tensors, multi-chunk tensors with a partial last chunk on either path, the
down4 conv weight of the ResUNet (320 x 256 x 27 = 270 full chunks), a non-finite gradient in the last chunk of the
largest tensor (inf or NaN), and a run without an EMA model."""
import pytest
import torch

pytestmark = pytest.mark.gpu

CHUNK = 8192
SMALL = [(33, 7, 3, 3, 3), (4096,), (5,), (128, 64, 1, 1, 1), (3, 1)]
# name: (shapes, overflow value, (tensor, flat index) of it or "last" = last element of the largest tensor, with EMA)
CASES = {
    "small": (SMALL, float("inf"), (1, 17), True),
    "float4_chunks": ([(3 * CHUNK + 4,), (5,)], float("inf"), "last", True),
    "scalar_chunks": ([(2 * CHUNK + 3,), (64, 32)], float("inf"), "last", True),
    "conv_270_chunks": ([(320, 256, 3, 3, 3), (320,)], float("inf"), "last", True),
    "nan_last_chunk": ([(3 * CHUNK + 4,), (2 * CHUNK + 3,)], float("nan"), "last", True),
    "no_ema": (SMALL, float("inf"), (1, 17), False),
}
# the original five-tensor set keeps its ids
PARAMS = [pytest.param("small", amp, id=str(amp)) for amp in (True, False)] + \
         [pytest.param(c, amp, id="%s-%s" % (c, amp)) for c in CASES if c != "small" for amp in (True, False)]


def _ema_reference(model_params, ema_params, alpha, global_step):
    alpha = min(1 - 1 / (global_step + 1), alpha)
    for e, p in zip(ema_params, model_params):
        e.data.mul_(alpha).add_(p.data, alpha=1 - alpha)      # training/utils.py:101-102


@pytest.mark.parametrize("case,amp", PARAMS)
def test_fused_adamw_ema_matches_torch(case, amp):
    from b200seg.train import FusedAdamWEMA
    torch.manual_seed(3)
    shapes, bad_value, where, with_ema = CASES[case]
    net = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(*s, device="cuda")) for s in shapes])
    ema = torch.nn.ParameterList([torch.nn.Parameter(p.detach().clone(), requires_grad=False) for p in net])
    ref = [p.detach().clone().requires_grad_(True) for p in net]
    ref_ema = [p.detach().clone() for p in net]
    ema0 = [e.detach().clone() for e in ema]
    opt = torch.optim.AdamW(ref, lr=1e-3, betas=(0.9, 0.999), weight_decay=0.05, eps=1e-5, fused=True)
    scaler = torch.amp.GradScaler("cuda", enabled=amp, init_scale=1024.0, growth_interval=3)
    fused = FusedAdamWEMA(net, ema if with_ema else None, lr=1e-3, amp=amp, init_scale=1024.0, growth_interval=3)
    if where == "last":
        big = max(range(len(shapes)), key=lambda i: net[i].numel())
        where = (big, net[big].numel() - 1)
    for it in range(7):
        grads = [torch.randn_like(p) * 0.1 for p in net]
        if amp and it == 2:
            grads[where[0]].view(-1)[where[1]] = bad_value           # an overflow step
        if amp:
            scaler.scale(torch.zeros(1, device="cuda"))      # lazily creates the scaler's device-side scale tensor
        scale = scaler.get_scale() if amp else 1.0
        for p, r, g in zip(net, ref, grads):
            p.grad = (g * scale).clone()
            r.grad = (g * scale).clone()
        fused.step()
        if amp:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        _ema_reference(ref, ref_ema, 0.99, it)
        if amp:
            assert abs(fused.scale.item() - scaler.get_scale()) < 1e-6, (it, fused.scale.item(), scaler.get_scale())
        for p, r in zip(net, ref):
            assert torch.allclose(p, r, rtol=2e-6, atol=1e-7), (it, (p - r).abs().max().item())
        for e, r, e0 in zip(ema, ref_ema, ema0):
            if with_ema:
                assert torch.allclose(e, r, rtol=2e-6, atol=1e-7), (it, (e - r).abs().max().item())
            else:
                assert torch.equal(e, e0)          # the table row carries no EMA pointer
    assert fused.step_dev.item() == (6 if amp else 7)
    assert fused._tables[2] == sum(-(-p.numel() // CHUNK) for p in net)      # chunks launched per step
