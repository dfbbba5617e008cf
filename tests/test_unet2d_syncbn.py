"""World size 2: the 2D UNet / ResUNet wrapped as train_ddp.py:352-358 does (SyncBatchNorm.convert_sync_batchnorm +
DistributedDataParallel) against the same network, with plain BatchNorm, run on the concatenated batch in one process:
  * each rank's BatchNorm statistics give its slice of the full-batch output,
  * every rank's running buffers (and num_batches_tracked) equal those of the full-batch run,
  * the DDP-reduced gradient (the mean over ranks of per-rank means) equals the full-batch gradient.
Over gloo on the CPU with the C-ABI ops emulated (tests/emu_bn.py), and over NCCL on two GPUs with the real kernels."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B_RANK, H = 2, 32


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, q, backend):
    try:
        q.put((rank, _compare(rank, world, port, backend)))
    except BaseException as e:          # report instead of leaving the other rank waiting
        q.put((rank, repr(e)))
        raise


def _compare(rank, world, port, backend):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    if backend == "nccl":
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
    else:
        dev = torch.device("cpu")
    dist.init_process_group(backend, rank=rank, world_size=world)
    import b200seg
    from oracle.make_golden_unet2d import batch, seeded_state_dict
    if backend == "gloo":
        import emu_bn

        class MP:
            def setattr(self, obj, name, val):
                setattr(obj, name, val)
        emu_bn.install(MP())
        torch.Tensor.is_cuda = property(lambda self: True)
    out = {}
    for block in ("SingleConv", "BasicBlock"):
        img, _ = batch(B_RANK * world, H, H, 4, seed=300)
        img = img.to(dev)
        wmap = torch.randn(1, 4, H, H, generator=torch.Generator().manual_seed(5)).to(dev)

        def build():
            net = b200seg.UNet2D(1, 4, 8, block=block)
            net.load_state_dict(seeded_state_dict(net, 11))
            return net.to(dev)

        # the full batch in one process, plain BatchNorm
        full = build()
        y_full = full(img)
        (y_full * wmap).mean().backward()
        # this rank's slice through the DDP-wrapped SyncBatchNorm model
        net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(build())
        assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in net.modules())
        mine = slice(rank * B_RANK, (rank + 1) * B_RANK)
        if backend == "nccl":
            ddp = torch.nn.parallel.DistributedDataParallel(net, device_ids=[rank], find_unused_parameters=True)
            y = ddp(img[mine])
            (y * wmap).mean().backward()
        else:
            # DDP refuses SyncBatchNorm in a CPU module, so the gloo run reduces the gradients the way DDP does
            y = net(img[mine])
            (y * wmap).mean().backward()
            for p in net.parameters():
                dist.all_reduce(p.grad)
                p.grad /= world

        def err(a, b):
            a, b = a.detach().double().cpu(), b.detach().double().cpu()
            return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()
        sd, sd_full = net.state_dict(), full.state_dict()
        gmax = max(pf.grad.abs().max() for pf in full.parameters())
        running = [k for k in sd if "running_" in k]
        out[block] = {
            "out": err(y, y_full[mine]),
            "running": max(err(sd[k], sd_full[k]) for k in running),
            "nbt": all(torch.equal(sd[k].cpu(), sd_full[k].cpu()) for k in sd if k.endswith("num_batches_tracked")),
            # relative to each tensor's largest gradient, but not below 1e-3 of the network's: conv_ch.bias of a
            # ResUNet feeds only BatchNorms, so its true gradient is 0 and both runs hold round-off there
            "grad": max(((p.grad - pf.grad).abs().max() / max(pf.grad.abs().max(), 1e-3 * gmax)).item()
                        for p, pf in zip(net.parameters(), full.parameters())),
        }
    dist.destroy_process_group()
    return out


def _run(backend, tol):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, backend)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(60)
    for rank, out in res.items():
        assert isinstance(out, dict), (rank, out)
        for block, e in out.items():
            assert e["nbt"], (rank, block)
            assert e["out"] < tol and e["running"] < tol and e["grad"] < tol, (rank, block, e)


def test_syncbn_gloo_world2_matches_full_batch():
    _run("gloo", 1e-4)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_syncbn_nccl_world2_matches_full_batch():
    _run("nccl", 5e-3)
