"""PEM RGB branch on H100 kernels (SURVEY.md 8f, row N1): drop-in for `ViT`, `ViT_AE` and `ViTEncoder` of
PEM/model/feature_extraction.py:17-181.

The reference subclasses timm's VisionTransformer (ViT-B/16, 224 x 224, cls token, learned 197-position embedding, pre-norm
blocks, LayerNorm eps 1e-6, GELU MLP x4), takes the normalised outputs of blocks 2/5/8/11, concatenates them (3072 channels),
applies `output_upscaling` Linear(3072 -> 16*256), reshapes to a (B,256,56,56) map, F.interpolate's it to (B,256,224,224)
and gathers the 2048 chosen pixels per image.  Here:
    patch embedding, qkv / proj / fc1 / fc2 / output_upscaling  -> sam6d_gemm_tma (wgmma; GELU, bias, residual in the epilogue;
                                                                   V^T of every attention layer written by the qkv epilogue)
    LayerNorm                                                   -> sam6d_layernorm_bf16 (fp32 residual stream -> bf16 operand)
    attention (197 tokens, 12 heads x 64)                       -> sam6d_attn_tc
    56x56 map + bilinear upsampling + pixel gather              -> sam6d_bilinear_gather straight from the Linear output
                                                                   (the 1.6 GB (B,256,224,224) tensor is never formed)
Parameter names follow timm (`cls_token`, `pos_embed`, `patch_embed.proj`, `blocks.N.{norm1,attn.{qkv,proj},norm2,mlp.{fc1,fc2}}`,
`norm`, `head`) so that `feature_extraction.rgb_net.vit.*` / `rgb_net.output_upscaling.*` of a SAM-6D PEM checkpoint load.
timm is neither vendored nor pinned by the reference and is absent here: parity of this module is pinned only against
oracle/vit_oracle.py (a restatement of timm's documented forward), see DESIGN.md section 3.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .layers import _W, _f32, _Packed, _PatchEmbed, _Attention, _Mlp, PRECISIONS, block, pack_block, patch_embed, patch_rows
from .pem import _cfg, sample_pts_feats


class _Block(nn.Module):
    def __init__(self, dim, mlp_ratio, qkv_bias, norm_layer):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = _Attention(dim, qkv_bias)
        self.norm2 = norm_layer(dim)
        self.mlp = _Mlp(dim, int(dim * mlp_ratio))


class ViT(nn.Module):
    """feature_extraction.py:17-35: forward(x (B,3,224,224)) -> [norm(x_after_block_i) for i in (d-1, d-n-1, d-2n-1, d-3n-1)],
    each (B, 1 + 14*14, embed_dim), in block order (shallowest first), like the reference's `out` list."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0, qkv_bias=True,
                 norm_layer=None, num_classes=1000, precision="bf16"):
        super().__init__()
        norm_layer = norm_layer or (lambda d: nn.LayerNorm(d, eps=1e-6))
        if embed_dim // num_heads != 64 or embed_dim % num_heads:
            raise ValueError("sam6d_b200 ViT: head_dim 64 (ViT-B: 768 / 12, ViT-L: 1024 / 16)")
        self.img_size, self.patch_size, self.embed_dim, self.num_heads, self.depth = img_size, patch_size, embed_dim, num_heads, depth
        self.patch_embed = _PatchEmbed(patch_size, in_chans, embed_dim)
        n_patches = (img_size // patch_size) ** 2
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.randn(1, n_patches + 1, embed_dim) * .02)
        self.blocks = nn.ModuleList([_Block(embed_dim, mlp_ratio, qkv_bias, norm_layer) for _ in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()   # unused, kept for the state_dict
        self.precision = precision
        self._packed = _Packed()

    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        C = self.embed_dim
        return dict(pe_w=_W(self.patch_embed.proj.weight.reshape(C, -1)), pe_b=_f32(self.patch_embed.proj.bias),
                    cls=(_f32(self.cls_token).reshape(C) + _f32(self.pos_embed)[0, 0]).contiguous(),
                    pos=_f32(self.pos_embed)[0, 1:].contiguous(), nw=_f32(self.norm.weight), nb=_f32(self.norm.bias),
                    neps=self.norm.eps,
                    blocks=[pack_block(blk.norm1, blk.attn.qkv.weight, blk.attn.qkv.bias, blk.attn.proj.weight, blk.attn.proj.bias,
                                       blk.norm2, blk.mlp.fc1.weight, blk.mlp.fc1.bias, blk.mlp.fc2.weight, blk.mlp.fc2.bias)
                            for blk in self.blocks])

    def _attend(self, bw, xn, B, S):
        C = self.embed_dim
        H, d = self.num_heads, C // self.num_heads
        if self.precision == "bf16":
            qk, vt = ops.gemm_tma_vt(xn, bw["qkv"].bf16, bw["qkv_b"], 2 * C, S, slot=3)
            return ops.attn_tc(qk, 0, qk, C, vt, B, H, S, S, d, d ** -0.5, out_dtype=torch.bfloat16)
        qkv = ops.gemm(xn, bw["qkv"].f32, bw["qkv_b"])
        att = torch.empty(B * S, C, dtype=torch.float32, device=xn.device)
        qkv = qkv.view(B, S, 3 * C)
        ops.mha(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], None, d ** -0.5, att.view(B, S, C))
        return att

    @torch.no_grad()
    def forward_tokens(self, x):
        """-> list of the four normalised outputs as (B*S, C) rows (bf16 in bf16 mode), plus (B, S)"""
        if not x.is_cuda:
            raise RuntimeError("sam6d_b200 ViT needs CUDA tensors: there is no CPU path")
        w = self._weights()
        B, Cin, Himg, Wimg = x.shape
        P, C = self.patch_size, self.embed_dim
        G = Himg // P
        L, S = G * G, G * G + 1
        if w["pos"].shape[0] != L:
            raise RuntimeError(f"pos_embed has {w['pos'].shape[0]} patch positions, the image gives {L}")
        rows = patch_rows(x, P)
        tok = torch.empty(B, S, C, dtype=torch.float32, device=x.device)
        tok[:, 0, :] = w["cls"]                                      # cls_token + pos_embed[0]
        # patch tokens = patches W^T + b + pos_embed[1:], written behind the cls row of every image
        patch_embed(self.precision, rows, w["pe_w"], w["pe_b"], w["pos"], tok[:, 1:, :])
        tok = tok.view(B * S, C)
        d = self.depth
        n = d // 4
        taps = (d - 1, d - n - 1, d - 2 * n - 1, d - 3 * n - 1)
        outs = []
        for idx, bw in enumerate(w["blocks"]):
            tok = block(self.precision, bw, tok, lambda xn: self._attend(bw, xn, B, S))
            if idx in taps:
                if self.precision == "bf16":
                    outs.append(ops.layernorm_bf16(tok, w["nw"], w["nb"], eps=w["neps"]))
                else:
                    outs.append(ops.layernorm(tok, w["nw"], w["nb"], eps=w["neps"]))
        return outs, B, S

    @torch.no_grad()
    def forward(self, x):
        outs, B, S = self.forward_tokens(x)
        return [o.float().view(B, S, self.embed_dim) for o in outs]


class ViT_AE(nn.Module):
    """feature_extraction.py:39-108 with up_type='linear' (PEM/config/base.yaml:19-25).  forward(x) -> (B,out_dim,H,W), cls."""

    def __init__(self, cfg, precision="bf16"):
        super().__init__()
        cfg = _cfg(cfg, vit_type="vit_base", up_type="linear", embed_dim=768, out_dim=256, use_pyramid_feat=True, pretrained=False)
        self.cfg = cfg
        if cfg.up_type != "linear":
            raise NotImplementedError("SAM-6D configures up_type='linear'")
        depth, heads = {"vit_base": (12, 12), "vit_large": (24, 16)}[cfg.vit_type]
        depth = getattr(cfg, "depth", depth)
        heads = getattr(cfg, "num_heads", heads)
        self.embed_dim, self.out_dim, self.use_pyramid_feat = cfg.embed_dim, cfg.out_dim, cfg.use_pyramid_feat
        self.vit = ViT(patch_size=16, embed_dim=cfg.embed_dim, depth=depth, num_heads=heads, mlp_ratio=4, qkv_bias=True,
                       img_size=getattr(cfg, "img_size", 224), precision=precision)
        nblock = 4 if cfg.use_pyramid_feat else 1
        self.output_upscaling = nn.Linear(cfg.embed_dim * nblock, 16 * cfg.out_dim, bias=True)
        self.precision = precision
        self._packed = _Packed()
        # (the reference downloads the MAE checkpoint when cfg.pretrained: weights come from load_state_dict here)

    def _weights(self):
        return self._packed.get(lambda: dict(up=_W(self.output_upscaling.weight), up_b=_f32(self.output_upscaling.bias)),
                                self.output_upscaling)

    @torch.no_grad()
    def upscaled_tokens(self, x):
        """output_upscaling(cat(pyramid)[:, 1:]) as (B, 196, 16*out_dim) (bf16 in bf16 mode) and the last level's cls tokens"""
        self.vit.precision = self.precision
        outs, B, S = self.vit.forward_tokens(x)
        C = self.embed_dim
        cls_tokens = outs[-1].view(B, S, C)[:, 0, :].float().contiguous()
        levels = outs if self.use_pyramid_feat else outs[-1:]
        feat = torch.cat([o.view(B, S, C)[:, 1:, :] for o in levels], dim=2).reshape(B * (S - 1), C * len(levels)).contiguous()
        w = self._weights()
        if self.precision == "bf16":
            up = ops.gemm_tma(feat, w["up"].bf16, w["up_b"], out_dtype=torch.bfloat16)
        else:
            up = ops.gemm(feat, w["up"].f32, w["up_b"])
        return up.view(B, S - 1, -1), cls_tokens

    @torch.no_grad()
    def forward(self, x):
        """the reference's contract: the full (B, out_dim, H, W) bilinear map (use ViTEncoder.get_img_feats on the hot path)"""
        B, _, H, W = x.shape
        up, cls_tokens = self.upscaled_tokens(x)
        G = int(math.isqrt(up.shape[1]))
        every = torch.arange(H * W, device=x.device, dtype=torch.int64).unsqueeze(0).expand(B, -1).contiguous()
        full = ops.bilinear_gather(up, every, G, 4, self.out_dim, H, W)
        return full.view(B, H, W, self.out_dim).permute(0, 3, 1, 2).contiguous(), cls_tokens


class ViTEncoder(nn.Module):
    """feature_extraction.py:113-181 (inference branch).  get_img_feats(img (B,3,224,224), choose (B,npoint) int64) -> (B,npoint,
    out_dim); get_obj_feats(...) builds the template bank; forward(end_points) -> (dense_pm, dense_fm, dense_po, dense_fo, radius)."""

    def __init__(self, cfg=None, npoint=2048, precision="bf16"):
        super().__init__()
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}")
        self.npoint = npoint
        self.rgb_net = ViT_AE(cfg if cfg is not None else SimpleNamespace(), precision=precision)
        self.precision = precision

    @torch.no_grad()
    def get_img_feats(self, img, choose):
        self.rgb_net.precision = self.precision
        B, _, H, W = img.shape
        up, _ = self.rgb_net.upscaled_tokens(img)
        G = int(math.isqrt(up.shape[1]))
        return ops.bilinear_gather(up, choose.contiguous(), G, 4, self.rgb_net.out_dim, H, W)

    @torch.no_grad()
    def get_obj_feats(self, tem_rgb_list, tem_pts_list, tem_choose_list, npoint=None):
        npoint = self.npoint if npoint is None else npoint
        feats = [self.get_img_feats(t, c) for t, c in zip(tem_rgb_list, tem_choose_list)]
        return sample_pts_feats(torch.cat(tem_pts_list, dim=1).contiguous(), torch.cat(feats, dim=1).contiguous(), npoint)

    @torch.no_grad()
    def forward(self, end_points):
        if self.training:
            raise NotImplementedError("sam6d_b200 implements the inference path (model.eval())")
        dense_fm = self.get_img_feats(end_points['rgb'], end_points['rgb_choose'])
        assert end_points['rgb_choose'].size(1) == self.npoint
        dense_po = end_points['dense_po'].contiguous()
        radius = ops.cloud_radius(dense_po)
        dense_pm = ops.scale_by_radius(end_points['pts'].contiguous(), radius)
        dense_po = ops.scale_by_radius(dense_po, radius)
        return dense_pm, dense_fm, dense_po, end_points['dense_fo'].clone(), radius
