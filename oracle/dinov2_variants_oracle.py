"""oracle/dinov2_variants_oracle.py -- TEST INFRASTRUCTURE ONLY.

CPU restatement (torch fp32) of the four DINOv2 descriptor backbones the reference's CustomDINOv2 maps its model names to
(ISM/model/dinov2.py:14-26; constructors ISM/model/vision_transformer.py:336-392).  dinov2_oracle.py restates ViT-L/14 with the
Mlp FFN; this module takes the architecture as arguments and adds the SwiGLU FFN of ViT-g/14:
    SwiGLUFFN.forward   ISM/model/layers/swiglu_ffn.py:29-33   (SwiGLUFFNFused :45-63 without xformers: hidden (int(4C*2/3)+7)//8*8)
Everything else (proposal preprocessing, pos-embed interpolation, the patch-validity rule) is dinov2_oracle's.
Parity status: PINNED -- tools/make_golden_dinov2_variants.py instantiates the reference's own vit_small / vit_base /
vit_giant2(ffn_layer="swiglufused"), loads the same seeded state dicts and finds this restatement bit-identical; fixture
tests/golden/dinov2_variants.pt."""
from typing import Dict

import torch
import torch.nn.functional as F

from oracle.dinov2_oracle import interpolate_pos_encoding, make_state_dict as _make_state_dict

SD = Dict[str, torch.Tensor]

# model name -> (embed_dim, num_heads, depth, ffn_layer).  ViT-g is built with the SwiGLU FFN its published checkpoint holds.
ARCHS = {
    "dinov2_vits14": (384, 6, 12, "mlp"),
    "dinov2_vitb14": (768, 12, 12, "mlp"),
    "dinov2_vitl14": (1024, 16, 24, "mlp"),
    "dinov2_vitg14": (1536, 24, 40, "swiglufused"),
}


def make_state_dict(model_name: str, seed: int = 1) -> SD:
    """seeded weights of `model_name` under the reference's key names (sam6d_b200.synth.make_dinov2_state_dict)"""
    C, heads, depth, ffn = ARCHS[model_name]
    return _make_state_dict(embed_dim=C, depth=depth, num_heads=heads, seed=seed, ffn_layer=ffn)


def vit_forward(sd: SD, x: torch.Tensor, num_heads: int, patch: int = 14, ffn: str = "mlp"):
    """DinoVisionTransformer.forward_features (vision_transformer.py:212-267) -> dict(x_norm_clstoken (B,C), x_norm_patchtokens (B,L,C))"""
    B, _, w, h = x.shape
    t = F.conv2d(x, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch).flatten(2).transpose(1, 2)
    t = torch.cat((sd["cls_token"].expand(B, -1, -1), t), dim=1)
    t = t + interpolate_pos_encoding(sd["pos_embed"], t.shape[1] - 1, w, h, patch)
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    C = t.shape[-1]
    hd = C // num_heads
    for i in range(depth):
        p = f"blocks.{i}."
        y = F.layer_norm(t, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
        qkv = F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, -1, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0] * hd ** -0.5, qkv[1], qkv[2]
        a = (q @ k.transpose(-2, -1)).softmax(dim=-1)
        y = (a @ v).transpose(1, 2).reshape(B, -1, C)
        y = F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        t = t + y * sd[p + "ls1.gamma"]
        y = F.layer_norm(t, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
        if ffn == "swiglufused":
            x1, x2 = F.linear(y, sd[p + "mlp.w12.weight"], sd[p + "mlp.w12.bias"]).chunk(2, dim=-1)
            y = F.linear(F.silu(x1) * x2, sd[p + "mlp.w3.weight"], sd[p + "mlp.w3.bias"])
        else:
            y = F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
        t = t + y * sd[p + "ls2.gamma"]
    n = F.layer_norm(t, (C,), sd["norm.weight"], sd["norm.bias"], 1e-6)
    return dict(x_norm_clstoken=n[:, 0], x_norm_patchtokens=n[:, 1:])


def cls_and_patch_features(sd: SD, images: torch.Tensor, masks: torch.Tensor, model_name: str, patch: int = 14, thresh: float = 0.5):
    """dinov2.py:248-258 for `model_name`: cls tokens (P,C); patch tokens masked by AvgPool2d(14)(mask) > 0.5, L2-normalised (P,L,C)"""
    _, heads, _, ffn = ARCHS[model_name]
    f = vit_forward(sd, images, heads, patch, ffn)
    keep = F.avg_pool2d(masks.unsqueeze(1), patch, patch).flatten(-2).squeeze(1) > thresh
    pf = F.normalize(f["x_norm_patchtokens"] * keep.unsqueeze(-1), dim=-1)
    return f["x_norm_clstoken"], pf, keep
