"""Pin oracle/unetr.py (whole-model functional restatement) against the reference's UNETR class and write
tests/golden/unetr_small.pt.

model/dim3/unetr.py is imported UNMODIFIED.  The `monai` symbols it pulls in (monai 1.1.0 is not installed and its source
is not part of the reference checkout) are working stand-ins written from MONAI 1.1.0's published semantics: the
SwinUNETR stand-ins of make_golden_swin_unetr.install_monai_standin (UnetrBasicBlock, UnetrUpBlock, UnetOutBlock) plus
ViT (PatchEmbeddingBlock, TransformerBlock, SABlock, MLPBlock) and UnetrPrUpBlock below, with MONAI's module names,
registration order and initialisation.  So this run pins UNETR.forward's wiring (which hidden states feed which
encoder, proj_feat) while the monai blocks stay "parity unpinned".
Runs only where the reference checkout is available (oracle/make_golden.py: B200SEG_REFERENCE).  Usage:  python oracle/make_golden_unetr.py
"""
import math
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import digest, import_reference     # noqa: E402
from oracle.make_golden_swin_unetr import install_monai_standin as install_swin_standin   # noqa: E402
from oracle import losses as olosses                         # noqa: E402
from oracle import unetr as ounetr                           # noqa: E402
from oracle.synth import make_volume                         # noqa: E402


def trunc_normal_(t, mean=0.0, std=1.0, a=-2.0, b=2.0):
    """monai PatchEmbeddingBlock.trunc_normal_: inverse-CDF sampling of a truncated normal."""
    def norm_cdf(x):
        return (1.0 + math.erf(x / math.sqrt(2.0))) / 2.0
    with torch.no_grad():
        lo, up = norm_cdf((a - mean) / std), norm_cdf((b - mean) / std)
        t.uniform_(2 * lo - 1, 2 * up - 1)
        t.erfinv_()
        t.mul_(std * math.sqrt(2.0))
        t.add_(mean)
        t.clamp_(min=a, max=b)
        return t


class Rearrange(nn.Module):
    def __init__(self, pattern, **axes):
        super().__init__()
        self.pattern, self.axes = pattern, axes

    def forward(self, x):
        return ounetr.patchify(x)


class PatchEmbeddingBlock(nn.Module):
    def __init__(self, in_channels, img_size, patch_size, hidden_size, num_heads, pos_embed, dropout_rate=0.0, spatial_dims=3):
        super().__init__()
        assert pos_embed == "perceptron" and spatial_dims == 3
        for m, p in zip(img_size, patch_size):
            if m % p != 0:
                raise ValueError("patch_size should be divisible by img_size for perceptron.")
        self.n_patches = int(torch.tensor([m // p for m, p in zip(img_size, patch_size)]).prod())
        self.patch_dim = int(in_channels * patch_size[0] * patch_size[1] * patch_size[2])
        self.patch_embeddings = nn.Sequential(Rearrange("b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)"),
                                              nn.Linear(self.patch_dim, hidden_size))
        self.position_embeddings = nn.Parameter(torch.zeros(1, self.n_patches, hidden_size))
        self.dropout = nn.Dropout(dropout_rate)
        trunc_normal_(self.position_embeddings, mean=0.0, std=0.02, a=-2.0, b=2.0)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, mean=0.0, std=0.02, a=-2.0, b=2.0)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, x):
        return self.dropout(self.patch_embeddings(x) + self.position_embeddings)


class MLPBlock(nn.Module):
    def __init__(self, hidden_size, mlp_dim, dropout_rate=0.0):
        super().__init__()
        self.linear1 = nn.Linear(hidden_size, mlp_dim)
        self.linear2 = nn.Linear(mlp_dim, hidden_size)
        self.fn = nn.GELU()
        self.drop1 = nn.Dropout(dropout_rate)
        self.drop2 = nn.Dropout(dropout_rate)

    def forward(self, x):
        return self.drop2(self.linear2(self.drop1(self.fn(self.linear1(x)))))


class SABlock(nn.Module):
    def __init__(self, hidden_size, num_heads, dropout_rate=0.0, qkv_bias=False):
        super().__init__()
        self.num_heads = num_heads
        self.out_proj = nn.Linear(hidden_size, hidden_size)
        self.qkv = nn.Linear(hidden_size, hidden_size * 3, bias=qkv_bias)
        self.drop_output = nn.Dropout(dropout_rate)
        self.drop_weights = nn.Dropout(dropout_rate)
        self.head_dim = hidden_size // num_heads
        self.scale = self.head_dim ** -0.5

    def forward(self, x):
        b, n, c = x.shape
        q, k, v = self.qkv(x).reshape(b, n, 3, self.num_heads, self.head_dim).permute(2, 0, 3, 1, 4)   # "b h (qkv l d) -> qkv b l h d"
        att = self.drop_weights((torch.einsum("blxd,blyd->blxy", q, k) * self.scale).softmax(dim=-1))
        x = torch.einsum("bhxy,bhyd->bhxd", att, v).permute(0, 2, 1, 3).reshape(b, n, c)            # "b h l d -> b l (h d)"
        return self.drop_output(self.out_proj(x))


class TransformerBlock(nn.Module):
    def __init__(self, hidden_size, mlp_dim, num_heads, dropout_rate=0.0, qkv_bias=False):
        super().__init__()
        self.mlp = MLPBlock(hidden_size, mlp_dim, dropout_rate)
        self.norm1 = nn.LayerNorm(hidden_size)
        self.attn = SABlock(hidden_size, num_heads, dropout_rate, qkv_bias)
        self.norm2 = nn.LayerNorm(hidden_size)

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class ViT(nn.Module):
    def __init__(self, in_channels, img_size, patch_size, hidden_size=768, mlp_dim=3072, num_layers=12, num_heads=12,
                 pos_embed="conv", classification=False, num_classes=2, dropout_rate=0.0, spatial_dims=3,
                 post_activation="Tanh", qkv_bias=False):
        super().__init__()
        if hidden_size % num_heads != 0:
            raise ValueError("hidden_size should be divisible by num_heads.")
        assert not classification
        self.classification = classification
        self.patch_embedding = PatchEmbeddingBlock(in_channels, img_size, patch_size, hidden_size, num_heads, pos_embed,
                                                   dropout_rate, spatial_dims)
        self.blocks = nn.ModuleList([TransformerBlock(hidden_size, mlp_dim, num_heads, dropout_rate, qkv_bias)
                                     for _ in range(num_layers)])
        self.norm = nn.LayerNorm(hidden_size)

    def forward(self, x):
        x = self.patch_embedding(x)
        hidden_states_out = []
        for blk in self.blocks:
            x = blk(x)
            hidden_states_out.append(x)
        return self.norm(x), hidden_states_out


class TranspConv(nn.Module):              # monai Convolution(is_transposed=True, conv_only=True, bias=False): child `conv`
    def __init__(self, ci, co):
        super().__init__()
        self.conv = nn.ConvTranspose3d(ci, co, kernel_size=2, stride=2, bias=False)

    def forward(self, x):
        return self.conv(x)


class UnetrPrUpBlock(nn.Module):
    def __init__(self, spatial_dims, in_channels, out_channels, num_layer, kernel_size, stride, upsample_kernel_size,
                 norm_name, conv_block=False, res_block=False):
        super().__init__()
        assert not conv_block and upsample_kernel_size == 2
        self.transp_conv_init = TranspConv(in_channels, out_channels)
        self.blocks = nn.ModuleList([TranspConv(out_channels, out_channels) for _ in range(num_layer)])

    def forward(self, x):
        x = self.transp_conv_init(x)
        for blk in self.blocks:
            x = blk(x)
        return x


def install_monai_standin():
    import types
    install_swin_standin()
    blocks = sys.modules["monai.networks.blocks"]
    blocks.UnetrPrUpBlock = UnetrPrUpBlock
    dyn = types.ModuleType("monai.networks.blocks.dynunet_block")
    dyn.UnetOutBlock = blocks.UnetOutBlock
    nets = types.ModuleType("monai.networks.nets")
    nets.ViT = ViT
    sys.modules.update({"monai.networks.blocks.dynunet_block": dyn, "monai.networks.nets": nets})


CASES = {  # name: (img size, in_ch, classes, feature_size, hidden, mlp, heads, ce weight, seeds)
    "unetr_small": ((32, 48, 64), 1, 3, 16, 128, 256, 2, [0.5, 1.0, 2.0], (81, 82)),
}


def main():
    torch.set_num_threads(8)
    import_reference()
    install_monai_standin()
    from model.dim3.unetr import UNETR
    out = os.path.join(ROOT, "tests", "golden")
    for name, (size, in_ch, classes, fs, hidden, mlp, heads, w, (sseed, dseed)) in CASES.items():
        net = UNETR(in_ch, classes, size, feature_size=fs, hidden_size=hidden, mlp_dim=mlp, num_heads=heads,
                    pos_embed="perceptron", norm_name="instance", res_block=True)
        keys = list(net.state_dict())
        shapes = ounetr.unetr_param_shapes(in_ch, classes, size, fs, hidden, mlp)
        assert keys == list(shapes), [k for k in keys if k not in shapes][:5] + [k for k in shapes if k not in keys][:5]
        for k in keys:
            assert tuple(net.state_dict()[k].shape) == shapes[k], k
        sd = ounetr.seeded_state_dict(shapes, sseed)
        net.load_state_dict(sd)
        img, lab = make_volume(2, *size, classes, seed=dseed, in_ch=in_ch)
        weight = torch.tensor(w)
        logits = net(img)
        loss = nn.CrossEntropyLoss(weight=weight)(logits, lab.squeeze(1)) + olosses.dice_loss(logits, lab)
        loss.backward()
        ref_grads = {k: p.grad.clone() for k, p in net.named_parameters()}
        so = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        lo = ounetr.unetr_forward(so, img, heads)
        lo_loss = olosses.total_loss(lo, lab, weight)
        lo_loss.backward()
        e = (lo - logits).abs().max().item() / logits.abs().max().item()
        print(name, "logits rel diff oracle vs reference class: %.2e, loss %.6f vs %.6f" % (e, lo_loss.item(), loss.item()))
        assert e < 1e-5 and abs(lo_loss.item() - loss.item()) < 1e-5
        worst = max(((so[k].grad - ref_grads[k]).abs().max() / (ref_grads[k].abs().max() + 1e-30)).item() for k in ref_grads)
        print(name, "worst grad rel diff %.2e over %d tensors (%d params)" % (worst, len(ref_grads), sum(v.numel() for v in sd.values())))
        assert worst < 2e-3
        torch.save({"cfg": dict(size=size, in_ch=in_ch, classes=classes, feature_size=fs, hidden=hidden, mlp=mlp, heads=heads,
                                batch=2, ce_weight=w, state_seed=sseed, data_seed=dseed),
                    "shapes": shapes, "logits": ounetr.voxel_sample(logits.detach()).half(),
                    "argmax": ounetr.voxel_sample(logits.detach()).argmax(1).to(torch.uint8), "stride": ounetr.FIXTURE_STRIDE,
                    "loss": loss.item(), "grad_digest": {k: {n: d[n] for n in ("sum", "abs", "sq")}
                                                          for k, d in ((k, digest(v)) for k, v in ref_grads.items())}},
                   os.path.join(out, name + ".pt"))


if __name__ == "__main__":
    main()
