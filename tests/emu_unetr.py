"""CPU emulation of the UNETR-specific C-ABI ops (TEST INFRASTRUCTURE, companion of emu_swin.py).

The autograd Functions of b200seg.unetr that talk to the library directly are replaced by plain-PyTorch stand-ins with
the same `apply` signature, written from the reference's semantics (monai's SABlock and PatchEmbeddingBlock), not from
the kernels; PosEmbedFn and DeriveWeightFn stay real (they only use the already-emulated copy_channels).  So the module
wiring of b200seg.UNETR (flat token view, batch boundaries in the token matrix, qkv channel order, which hidden states
feed which encoder, the depth<->space shuffles) runs end to end on the CPU."""
import emu_swin
from oracle import unetr as ounetr


def install(monkeypatch):
    sw = emu_swin.install(monkeypatch)
    from b200seg import unetr as ur

    class AttentionFn:
        @staticmethod
        def apply(qkv, B, heads):
            C3 = qkv.shape[-1]
            out = ounetr.sa_core(qkv.reshape(B, -1, C3), heads)
            return out.reshape(*qkv.shape[:-1], C3 // 3)

    class PatchifyFn:
        """Rearrange 'b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)' on the channels-last volume"""
        @staticmethod
        def apply(x):
            B, D, H, W, C = x.shape
            P = ounetr.PATCH
            return ounetr.patchify(x.permute(0, 4, 1, 2, 3)).reshape(B, D // P, H // P, W // P, P ** 3 * C)

    for name, cls in dict(AttentionFn=AttentionFn, PatchifyFn=PatchifyFn, DepthSpaceFn=sw.DepthSpaceFn).items():
        monkeypatch.setattr(ur, name, cls)
    return ur
