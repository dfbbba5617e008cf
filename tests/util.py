import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

POISON = 1000.0        # finite: an over-read multiplied by a zero weight must not turn into a false NaN failure
SENTINEL = -777.0      # exact in fp16


def wide(dense, ld, coff):
    """dense [..., C] as channels coff .. coff+C of a [..., ld] buffer whose other channels hold +-POISON."""
    C = dense.shape[-1]
    assert coff + C <= ld
    sign = 1.0 - 2.0 * (torch.arange(ld, device=dense.device) % 2)
    buf = (POISON * sign).to(dense.dtype).expand(*dense.shape[:-1], ld).contiguous()
    buf[..., coff:coff + C] = dense
    return buf


def sentinel(lead, ld, dtype):
    return torch.full((*lead, ld), SENTINEL, dtype=dtype, device="cuda")


def assert_untouched(buf, coff, C):
    """the channels of an output buffer outside its slice still hold the sentinel, bit for bit"""
    keep = torch.ones(buf.shape[-1], dtype=torch.bool, device=buf.device)
    keep[coff:coff + C] = False
    out = buf[..., keep]
    assert torch.equal(out, torch.full_like(out, SENTINEL))


def rel_err(a, b):
    """max-norm relative error: ||a-b||_inf / ||b||_inf (the parity metric of SURVEY.md §8d)."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def launched_kernels(module, fn, *args):
    """Names of the kernels `module.fn(*args)` launches (module: a test module; args: literals), recorded by
    torch.profiler in a Python process of its own.  A profiling session late in a long pytest process can lose launches,
    and each session makes that likelier for the next; in a fresh process the record is complete and the test process
    is left as it was."""
    return launched_kernels_each(module, [(fn, args)])[0]


def launched_kernels_each(module, calls):
    """launched_kernels for several (fn, args) calls of one module, one profiling session each, in one fresh process"""
    code = ("from torch.profiler import ProfilerActivity, profile\n"
            "out = []\n"
            "for fn, args in %r:\n"
            "    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:\n"
            "        getattr(m, fn)(*args)\n"
            "        torch.cuda.synchronize()\n"
            "    out.append(sorted({e.name for e in prof.events()}))\n") % [(f, tuple(a)) for f, a in calls]
    return _fresh(module, code)


def run_fresh(module, fn, *args):
    """module.fn(*args) (args: literals) in a Python process of its own; returns its JSON-serialisable result.  For
    whole-model steps whose allocations and autograd state should not stay in the test process."""
    return _fresh(module, "out = m.%s(*%r)\n" % (fn, tuple(args)))


def _fresh(module, body):
    import json
    import subprocess
    import sys
    code = ("import json, sys\n"
            "sys.path[:0] = [%r, %r]\n"
            "import torch\n"
            "import %s as m\n"
            "%s"
            "print(json.dumps(out))\n") % (os.path.join(ROOT, "tests"), ROOT, module, body)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=200)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)


def dice_per_class(a, b, C):
    """metric/utils.py:62-82 style one-hot Dice between two label maps."""
    out = []
    for c in range(C):
        x, y = (a == c), (b == c)
        den = x.sum().item() + y.sum().item()
        out.append(1.0 if den == 0 else 2.0 * (x & y).sum().item() / den)
    return out


def grad_noise_floor(sd, img, lab, weight, cfg):
    """Gradients of the reference-pinned oracle in fp64 (the exact answer) and the distance of the fp32
    evaluation (= the reference's own numbers, tests/golden) from it.  ReLU'(0) is discontinuous, so two valid
    fp32 evaluations differ wherever a pre-activation is within rounding of 0, and InstanceNorm spreads each
    such flip over a whole channel: this distance is the noise floor of "matches the reference's backward"."""
    from oracle import losses as olosses
    from oracle import unet3d as ounet
    out = {}
    for dt in (torch.float32, torch.float64):
        s = {k: v.to(dt).clone().requires_grad_(True) for k, v in sd.items()}
        lo = ounet.unet_forward(s, img.to(dt), cfg["scale"], cfg["kernel"], cfg["block"])
        olosses.total_loss(lo, lab, weight.to(dt)).backward()
        out[dt] = ({k: v.grad.double() for k, v in s.items()}, lo.detach().double())
    g32, g64 = out[torch.float32][0], out[torch.float64][0]
    floor_max = max(rel_err(g32[k], g64[k]) for k in g64)
    return g64, out[torch.float64][1], floor_max, global_l2(g32, g64)


def global_l2(ga, gb):
    num = sum(((ga[k].double().cpu() - gb[k].double().cpu()) ** 2).sum().item() for k in gb)
    den = sum((gb[k].double().cpu() ** 2).sum().item() for k in gb)
    return (num / den) ** 0.5
