"""ORACLE (test infrastructure — never imported by the product path): UNETR as one pure function of a state_dict.

The wiring follows the reference file and is pinned to it (oracle/make_golden_unetr.py):
  UNETR.forward                model/dim3/unetr.py:218-237 (hidden states 3 / 6 / 9 feed encoders 2-4, the final
                               vit.norm output feeds decoder5; proj_feat :189-193)
The monai 1.1.0 blocks it imports are not part of the reference checkout; they are restated from MONAI 1.1.0's published
semantics — "PARITY UNPINNED" for exactly these pieces:
  ViT               patch_embedding -> 12 TransformerBlocks (each output kept) -> LayerNorm
  PatchEmbeddingBlock(pos_embed='perceptron')  Rearrange 'b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)',
                    Linear, + position_embeddings [1, L, hidden]
  TransformerBlock  x + SABlock(norm1(x)), then x + MLPBlock(norm2(x))
  SABlock           qkv Linear (no bias), 'b h (qkv l d) -> qkv b l h d', softmax(q k^T * dh^-0.5) v,
                    'b h l d -> b l (h d)', out_proj Linear
  UnetrPrUpBlock(conv_block=False)  ConvTranspose3d(k2, s2, no bias) transp_conv_init, then num_layer more
Shared with the SwinUNETR oracle: UnetrBasicBlock / UnetResBlock, UnetrUpBlock, UnetOutBlock (oracle/swin_unetr.py).
"""
import torch
import torch.nn.functional as F

from .swin_unetr import res_block, up_block

PATCH = 16
NUM_LAYERS = 12


def sa_core(qkv, heads):
    """SABlock.forward between its Linears: qkv [b, n, 3*C] -> [b, n, C]."""
    b, n, c3 = qkv.shape
    C = c3 // 3
    q, k, v = qkv.reshape(b, n, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    att = (torch.einsum("blxd,blyd->blxy", q, k) * (C // heads) ** -0.5).softmax(dim=-1)
    return torch.einsum("bhxy,bhyd->bhxd", att, v).permute(0, 2, 1, 3).reshape(b, n, C)


def transformer_block(sd, pre, x, heads):
    c = x.shape[-1]
    h = F.layer_norm(x, (c,), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"])
    h = sa_core(F.linear(h, sd[pre + "attn.qkv.weight"], sd.get(pre + "attn.qkv.bias")), heads)
    x = x + F.linear(h, sd[pre + "attn.out_proj.weight"], sd[pre + "attn.out_proj.bias"])
    h = F.layer_norm(x, (c,), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"])
    h = F.linear(F.gelu(F.linear(h, sd[pre + "mlp.linear1.weight"], sd[pre + "mlp.linear1.bias"])),
                 sd[pre + "mlp.linear2.weight"], sd[pre + "mlp.linear2.bias"])
    return x + h


def patchify(x):
    """Rearrange 'b c (h p1) (w p2) (d p3) -> b (h w d) (p1 p2 p3 c)'."""
    b, c, D, H, W = x.shape
    P = PATCH
    t = x.reshape(b, c, D // P, P, H // P, P, W // P, P).permute(0, 2, 4, 6, 3, 5, 7, 1)
    return t.reshape(b, (D // P) * (H // P) * (W // P), P ** 3 * c)


def vit(sd, x, heads):
    """monai ViT (classification=False): returns (norm(last), [output of every block])."""
    t = F.linear(patchify(x), sd["vit.patch_embedding.patch_embeddings.1.weight"],
                 sd["vit.patch_embedding.patch_embeddings.1.bias"]) + sd["vit.patch_embedding.position_embeddings"]
    hs = []
    for i in range(NUM_LAYERS):
        t = transformer_block(sd, "vit.blocks.%d." % i, t, heads)
        hs.append(t)
    return F.layer_norm(t, (t.shape[-1],), sd["vit.norm.weight"], sd["vit.norm.bias"]), hs


def pr_up_block(sd, pre, x, num_layer):
    x = F.conv_transpose3d(x, sd[pre + "transp_conv_init.conv.weight"], stride=2)
    for i in range(num_layer):
        x = F.conv_transpose3d(x, sd[pre + "blocks.%d.conv.weight" % i], stride=2)
    return x


def unetr_forward(sd, x, heads):
    """x [B, in_ch, D, H, W] -> logits [B, classes, D, H, W]."""
    feat = tuple(s // PATCH for s in x.shape[2:])
    last, hs = vit(sd, x, heads)

    def proj_feat(t):
        return t.view(t.shape[0], *feat, t.shape[-1]).permute(0, 4, 1, 2, 3).contiguous()
    enc1 = res_block(sd, "encoder1.layer.", x)
    enc2 = pr_up_block(sd, "encoder2.", proj_feat(hs[3]), 2)
    enc3 = pr_up_block(sd, "encoder3.", proj_feat(hs[6]), 1)
    enc4 = pr_up_block(sd, "encoder4.", proj_feat(hs[9]), 0)
    dec3 = up_block(sd, "decoder5.", proj_feat(last), enc4)
    dec2 = up_block(sd, "decoder4.", dec3, enc3)
    dec1 = up_block(sd, "decoder3.", dec2, enc2)
    out = up_block(sd, "decoder2.", dec1, enc1)
    return F.conv3d(out, sd["out.conv.conv.weight"], sd["out.conv.conv.bias"])


def unetr_param_shapes(in_ch, classes, img_size, fs=16, hidden=768, mlp=3072):
    """state_dict key -> shape in registration order (vit, encoder1..4, decoder5..2, out)."""
    out = {}
    n = 1
    for s in img_size:
        n *= s // PATCH
    out["vit.patch_embedding.position_embeddings"] = (1, n, hidden)
    out["vit.patch_embedding.patch_embeddings.1.weight"] = (hidden, PATCH ** 3 * in_ch)
    out["vit.patch_embedding.patch_embeddings.1.bias"] = (hidden,)
    for i in range(NUM_LAYERS):
        b = "vit.blocks.%d." % i
        out[b + "mlp.linear1.weight"] = (mlp, hidden); out[b + "mlp.linear1.bias"] = (mlp,)
        out[b + "mlp.linear2.weight"] = (hidden, mlp); out[b + "mlp.linear2.bias"] = (hidden,)
        out[b + "norm1.weight"] = (hidden,); out[b + "norm1.bias"] = (hidden,)
        out[b + "attn.out_proj.weight"] = (hidden, hidden); out[b + "attn.out_proj.bias"] = (hidden,)
        out[b + "attn.qkv.weight"] = (3 * hidden, hidden)
        out[b + "norm2.weight"] = (hidden,); out[b + "norm2.bias"] = (hidden,)
    out["vit.norm.weight"] = (hidden,); out["vit.norm.bias"] = (hidden,)

    def res(pre, ci, co):
        out[pre + "conv1.conv.weight"] = (co, ci, 3, 3, 3)
        out[pre + "conv2.conv.weight"] = (co, co, 3, 3, 3)
        if ci != co:
            out[pre + "conv3.conv.weight"] = (co, ci, 1, 1, 1)
    res("encoder1.layer.", in_ch, fs)
    for name, co, nl in (("encoder2.", 2 * fs, 2), ("encoder3.", 4 * fs, 1), ("encoder4.", 8 * fs, 0)):
        out[name + "transp_conv_init.conv.weight"] = (hidden, co, 2, 2, 2)
        for i in range(nl):
            out[name + "blocks.%d.conv.weight" % i] = (co, co, 2, 2, 2)
    for name, ci, co in (("decoder5.", hidden, 8 * fs), ("decoder4.", 8 * fs, 4 * fs), ("decoder3.", 4 * fs, 2 * fs),
                         ("decoder2.", 2 * fs, fs)):
        out[name + "transp_conv.conv.weight"] = (ci, co, 2, 2, 2)
        res(name + "conv_block.", 2 * co, co)
    out["out.conv.conv.weight"] = (classes, fs, 1, 1, 1)
    out["out.conv.conv.bias"] = (classes,)
    return out


FIXTURE_STRIDE = 15


def voxel_sample(logits, stride=FIXTURE_STRIDE):
    """logits [B, C, D, H, W] -> the class vectors of every stride-th voxel in (B, D, H, W) order, [N, C]: what the
    whole-model fixture stores (a fixed 1/15 of the voxels keeps it small)."""
    return logits.permute(0, 2, 3, 4, 1).reshape(-1, logits.shape[1])[::stride]


def seeded_state_dict(shapes, seed):
    """make_state_dict with LayerNorm weights around 1 and a position table in [-0.5, 0.5] (shared by the fixture
    writer and the tests)."""
    from .unet3d import make_state_dict
    sd = make_state_dict(shapes, seed=seed)
    for k in sd:
        if k.endswith("norm1.weight") or k.endswith("norm2.weight") or k.endswith("norm.weight"):
            sd[k] = 1.0 + 0.1 * sd[k] / sd[k].abs().max()
        if k.endswith("position_embeddings"):
            sd[k] = 0.5 * sd[k] / sd[k].abs().max()
    return sd
