"""SAM ViT image encoder on H100 kernels -- drop-in for `segment_anything.modeling.image_encoder.ImageEncoderViT`
(ISM/segment_anything/modeling/image_encoder.py:17-116; built by ISM/segment_anything/build_sam.py:55-80 and reached through
`SamPredictor.set_image -> model.image_encoder(x)`, ISM/segment_anything/predictor.py:89).

All three SAM backbones of build_sam.py:14-46 are covered (VIT_CONFIGS, build_image_encoder): ViT-H (head dim 80), ViT-L and
ViT-B (head dim 64); the attention kernels are instantiated for exactly these two head dims.  Same constructor signature, same
parameter names (so `sam_vit_{h,l,b}_*.pth: image_encoder.*` load unchanged), same forward contract: (B,3,1024,1024) normalised
image -> (B,256,64,64).  The torch sub-modules are parameter containers; the
forward runs sm_90a kernels through the C ABI.  precision="bf16" (default):
    every Linear (qkv, proj, MLP)        -> sam6d_gemm_tma (persistent TMA-fed wgmma GEMM; GELU / bias / fp32 residual in the
                                            epilogue; the qkv projection writes V^T itself, sam6d_gemm_tma_vt)
    LayerNorm                            -> sam6d_layernorm_bf16 (fp32 residual stream -> bf16 GEMM operand)
    window partition (pad 64 -> 70 AFTER norm1) / unpartition -> sam6d_gather_rows with a static index map (-1 = zero pad row)
    windowed attention (14 x 14 tokens)  -> sam6d_attn_tc with the decomposed rel-pos bias (tables from two extra MMAs)
    global attention (64 x 64 tokens)    -> sam6d_attn_global_tc_ex (online softmax, scores never leave registers)
    patch embed 16x16/16, neck 1x1 and 3x3 (9 shifted GEMMs) -> sam6d_gemm_bf16 / sam6d_gemm_tma, LayerNorm2d -> sam6d_layernorm
precision="fp32" keeps everything on the CUDA-core kernels (sam6d_gemm_f32, sam6d_attn_relpos: flash-style, no HW x HW score
tensor) and is the exact-parity comparator (max error 8e-6 against the reference module).
"""
from typing import Optional, Tuple, Type

import torch
import torch.nn as nn

from . import ops
from .layers import _W, _f32, _gemm, _Packed, PRECISIONS, block, pack_block, patch_embed, patch_rows

HEAD_DIMS = (64, 80)            # the head dims sam6d_attn_relpos / sam6d_attn_global_tc_ex / sam6d_attn_tc are built for

# build_sam.py:14-46: embed_dim, depth, num_heads, global_attn_indexes per backbone (the keyword arguments of
# synth.make_sam_state_dict as well)
VIT_CONFIGS = {
    "vit_h": dict(embed_dim=1280, depth=32, num_heads=16, global_attn_indexes=(7, 15, 23, 31)),
    "vit_l": dict(embed_dim=1024, depth=24, num_heads=16, global_attn_indexes=(5, 11, 17, 23)),
    "vit_b": dict(embed_dim=768, depth=12, num_heads=12, global_attn_indexes=(2, 5, 8, 11)),
}


class LayerNorm2d(nn.Module):
    """ISM/segment_anything/modeling/common.py:31-43 (parameters only; evaluated channel-last by sam6d_layernorm)"""

    def __init__(self, num_channels: int, eps: float = 1e-6) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.ones(num_channels))
        self.bias = nn.Parameter(torch.zeros(num_channels))
        self.eps = eps


class MLPBlock(nn.Module):
    def __init__(self, embedding_dim: int, mlp_dim: int, act: Type[nn.Module] = nn.GELU) -> None:
        super().__init__()
        if act is not nn.GELU:
            raise ValueError("sam6d_b200 MLPBlock fuses nn.GELU (erf) in the GEMM epilogue")
        self.lin1 = nn.Linear(embedding_dim, mlp_dim)
        self.lin2 = nn.Linear(mlp_dim, embedding_dim)


class Attention(nn.Module):
    def __init__(self, dim, num_heads=8, qkv_bias=True, use_rel_pos=False, rel_pos_zero_init=True, input_size=None):
        super().__init__()
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.use_rel_pos = use_rel_pos
        if not use_rel_pos:
            raise ValueError("sam6d_b200 implements the SAM configuration (use_rel_pos=True)")
        assert input_size is not None
        self.input_size = input_size
        self.rel_pos_h = nn.Parameter(torch.zeros(2 * input_size[0] - 1, dim // num_heads))
        self.rel_pos_w = nn.Parameter(torch.zeros(2 * input_size[1] - 1, dim // num_heads))


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=True, norm_layer=nn.LayerNorm, act_layer=nn.GELU,
                 use_rel_pos=False, rel_pos_zero_init=True, window_size=0, input_size=None):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, use_rel_pos=use_rel_pos,
                              rel_pos_zero_init=rel_pos_zero_init,
                              input_size=input_size if window_size == 0 else (window_size, window_size))
        self.norm2 = norm_layer(dim)
        self.mlp = MLPBlock(embedding_dim=dim, mlp_dim=int(dim * mlp_ratio), act=act_layer)
        self.window_size = window_size


class PatchEmbed(nn.Module):
    def __init__(self, kernel_size=(16, 16), stride=(16, 16), padding=(0, 0), in_chans=3, embed_dim=768):
        super().__init__()
        if tuple(kernel_size) != tuple(stride) or tuple(padding) != (0, 0):
            raise ValueError("sam6d_b200 PatchEmbed: non-overlapping patches (kernel == stride, no padding)")
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=kernel_size, stride=stride, padding=padding)


class ImageEncoderViT(nn.Module):
    def __init__(self, img_size: int = 1024, patch_size: int = 16, in_chans: int = 3, embed_dim: int = 768, depth: int = 12,
                 num_heads: int = 12, mlp_ratio: float = 4.0, out_chans: int = 256, qkv_bias: bool = True,
                 norm_layer: Type[nn.Module] = nn.LayerNorm, act_layer: Type[nn.Module] = nn.GELU, use_abs_pos: bool = True,
                 use_rel_pos: bool = False, rel_pos_zero_init: bool = True, window_size: int = 0,
                 global_attn_indexes: Tuple[int, ...] = (), precision: str = "bf16") -> None:
        super().__init__()
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}")
        if embed_dim % num_heads or (embed_dim // num_heads) not in HEAD_DIMS:
            raise ValueError(f"the SAM attention kernels are built for head dims {HEAD_DIMS} (ViT-B 768 / 12, ViT-L 1024 / 16, "
                             f"ViT-H 1280 / 16); got embed_dim {embed_dim} / num_heads {num_heads}")
        self.img_size, self.patch_size, self.embed_dim, self.num_heads = img_size, patch_size, embed_dim, num_heads
        self.precision = precision
        self.patch_embed = PatchEmbed(kernel_size=(patch_size, patch_size), stride=(patch_size, patch_size), in_chans=in_chans,
                                      embed_dim=embed_dim)
        self.pos_embed: Optional[nn.Parameter] = None
        if use_abs_pos:
            self.pos_embed = nn.Parameter(torch.zeros(1, img_size // patch_size, img_size // patch_size, embed_dim))
        self.blocks = nn.ModuleList()
        for i in range(depth):
            self.blocks.append(Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, norm_layer=norm_layer,
                                     act_layer=act_layer, use_rel_pos=use_rel_pos, rel_pos_zero_init=rel_pos_zero_init,
                                     window_size=window_size if i not in global_attn_indexes else 0,
                                     input_size=(img_size // patch_size, img_size // patch_size)))
        self.neck = nn.Sequential(nn.Conv2d(embed_dim, out_chans, kernel_size=1, bias=False), LayerNorm2d(out_chans),
                                  nn.Conv2d(out_chans, out_chans, kernel_size=3, padding=1, bias=False), LayerNorm2d(out_chans))
        self._packed = _Packed()
        self._maps = {}

    # ------------------------------------------------------------------------------------------------------------ weights
    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        w = dict(pe_w=_W(self.patch_embed.proj.weight.reshape(self.embed_dim, -1)), pe_b=_f32(self.patch_embed.proj.bias),
                 pos=_f32(self.pos_embed).reshape(-1, self.embed_dim) if self.pos_embed is not None else None, blocks=[])
        for blk in self.blocks:
            a = blk.attn
            bw = pack_block(blk.norm1, a.qkv.weight, a.qkv.bias, a.proj.weight, a.proj.bias,
                            blk.norm2, blk.mlp.lin1.weight, blk.mlp.lin1.bias, blk.mlp.lin2.weight, blk.mlp.lin2.bias)
            bw.update(rh=_f32(a.rel_pos_h), rw=_f32(a.rel_pos_w),
                      rel_blob=(ops.pack_rel_pos(_f32(a.rel_pos_h), _f32(a.rel_pos_w), slab_rows=32 if a.rel_pos_h.shape[0] <= 32 else 128)
                                if a.rel_pos_h.shape[0] <= 128 and a.rel_pos_h.is_cuda else None))
            w["blocks"].append(bw)
        oc = self.neck[0].out_channels
        w["neck0"] = _W(self.neck[0].weight.reshape(oc, -1))
        w["ln1"] = (_f32(self.neck[1].weight), _f32(self.neck[1].bias), self.neck[1].eps)
        # 3x3 conv as 9 shifted 1x1 GEMMs: tap (kh,kw) -> weight[:, :, kh, kw]
        w["neck2"] = [_W(self.neck[2].weight[:, :, kh, kw]) for kh in range(3) for kw in range(3)]
        w["ln2"] = (_f32(self.neck[3].weight), _f32(self.neck[3].bias), self.neck[3].eps)
        return w

    # ------------------------------------------------------------------------------------------------------------ index maps
    def _index_maps(self, B: int, G: int, ws: int, device):
        """static gather maps: window partition with zero padding (window_partition, image_encoder.py:243-264), its inverse
        (window_unpartition :267-290), and the 9 shifted neighbourhoods of the 3x3 neck conv (padding=1)"""
        key = (B, G, ws, str(device))
        if key not in self._maps:
            Gp = ((G + ws - 1) // ws) * ws
            nwin = Gp // ws
            hh, ww = torch.meshgrid(torch.arange(Gp), torch.arange(Gp), indexing="ij")
            src = torch.where((hh < G) & (ww < G), hh * G + ww, torch.full_like(hh, -1))               # (Gp,Gp) padded grid
            part = src.view(nwin, ws, nwin, ws).permute(0, 2, 1, 3).reshape(-1)                          # (nwin*nwin*ws*ws)
            h, w_ = torch.meshgrid(torch.arange(G), torch.arange(G), indexing="ij")
            unpart = ((h // ws) * nwin + (w_ // ws)) * ws * ws + (h % ws) * ws + (w_ % ws)
            taps = []
            for dh in (-1, 0, 1):
                for dw in (-1, 0, 1):
                    nh, nw_ = h + dh, w_ + dw
                    ok = (nh >= 0) & (nh < G) & (nw_ >= 0) & (nw_ < G)
                    taps.append(torch.where(ok, nh * G + nw_, torch.full_like(nh, -1)).reshape(-1))
            mk = lambda t: t.to(torch.int32).unsqueeze(0).expand(B, -1).contiguous().to(device)   # noqa: E731
            self._maps[key] = dict(part=mk(part), unpart=mk(unpart.reshape(-1)), taps=[mk(t) for t in taps], nwin=nwin)
        return self._maps[key]

    # ------------------------------------------------------------------------------------------------------------ forward
    def _attend(self, blk, bw, xn, B, G, maps):
        """window partition (pad 64 -> 70 after norm1), relative-position attention, unpartition (drops the padded tokens;
        proj is token-wise, so it runs after it).  bf16: the tensor cores read bf16 operands and attention writes bf16."""
        C, nH = self.embed_dim, self.num_heads
        bf16 = self.precision == "bf16"
        gather = ops.gather_rows_bf16 if bf16 else ops.gather_rows
        if blk.window_size > 0:
            xn = gather(xn.view(B, G * G, C), maps["part"]).view(-1, C)                        # zero rows at the padding
            nW, Hs = B * maps["nwin"] * maps["nwin"], blk.window_size
        else:
            nW, Hs = B, G
        if not bf16:
            qkv = ops.gemm(xn, bw["qkv"].f32, bw["qkv_b"])
            att = ops.attn_relpos(qkv, nW, Hs, Hs, nH, bw["rh"], bw["rw"], blk.attn.scale)
        elif Hs * Hs <= 256:
            # windowed blocks: tensor-core attention (QK^T and PV on wgmma, decomposed rel-pos bias in the softmax warps)
            qk, vt = ops.gemm_tma_vt(xn, bw["qkv"].bf16, bw["qkv_b"], 2 * C, Hs * Hs)                   # [q|k] rows and V^T per window
            att = ops.attn_tc(qk, 0, qk, C, vt, nW, nH, Hs * Hs, Hs * Hs, C // nH, blk.attn.scale,
                              rel=(bw["rel_blob"], Hs, Hs), out_dtype=torch.bfloat16)
        elif Hs == 64 and bw["rel_blob"] is not None:
            # global blocks of the 64 x 64 grid (4096 keys): wgmma attention with an online softmax, scores never leave registers
            qk, vt = ops.gemm_tma_vt(xn, bw["qkv"].bf16, bw["qkv_b"], 2 * C, Hs * Hs, slot=2)
            att = ops.attn_global_tc(qk, vt, bw["rel_blob"], nW, nH, Hs, blk.attn.scale, D=C // nH)
        else:
            # other grids: flash-style CUDA-core kernel with online softmax
            qkv = ops.gemm_tma(xn, bw["qkv"].bf16, bw["qkv_b"])
            att = ops.attn_relpos(qkv, nW, Hs, Hs, nH, bw["rh"], bw["rw"], blk.attn.scale, out_dtype=torch.bfloat16)
        if blk.window_size > 0:
            att = gather(att.view(B, -1, C), maps["unpart"]).view(-1, C)
        return att

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("ImageEncoderViT (sam6d_b200) needs CUDA tensors: there is no CPU path")
        w = self._weights()
        prec = self.precision
        B, Cin, Himg, Wimg = x.shape
        P, C = self.patch_size, self.embed_dim
        G = Himg // P
        L = G * G
        # PatchEmbed (image_encoder.py:364-395): non-overlapping conv == GEMM over (c, kh, kw)-flattened patches; + pos_embed
        rows = patch_rows(x, P)
        if w["pos"] is not None:
            tok = torch.empty(B * L, C, dtype=torch.float32, device=x.device)
            patch_embed(prec, rows, w["pe_w"], w["pe_b"], w["pos"], tok.view(B, L, C))
        else:
            tok = _gemm(prec, rows, w["pe_w"], w["pe_b"])
        ws = max((b.window_size for b in self.blocks), default=0) or 14
        maps = self._index_maps(B, G, ws, x.device)
        for blk, bw in zip(self.blocks, w["blocks"]):
            tok = block(prec, bw, tok, lambda xn: self._attend(blk, bw, xn, B, G, maps))
        # neck (image_encoder.py:88-104)
        y = _gemm(prec, tok, w["neck0"])
        y = ops.layernorm(y, w["ln1"][0], w["ln1"][1], eps=w["ln1"][2])
        oc = y.shape[1]
        acc = None
        y3 = y.view(B, L, oc)
        for tap, Wt in zip(maps["taps"], w["neck2"]):
            shifted = ops.gather_rows(y3, tap).view(-1, oc)
            acc = _gemm(prec, shifted, Wt, None, residual=acc)
        out = ops.layernorm(acc, w["ln2"][0], w["ln2"][1], eps=w["ln2"][2])
        return out.view(B, G, G, oc).permute(0, 3, 1, 2).contiguous()


def build_image_encoder(name: str = "vit_h", precision: str = "bf16") -> ImageEncoderViT:
    """the image_encoder argument of ISM/segment_anything/build_sam.py:14-46,55-80 for `vit_h` (the variant SAM-6D's
    ISM/configs/model/segmentor_model/sam.yaml selects), `vit_l` or `vit_b`"""
    from functools import partial
    if name not in VIT_CONFIGS:
        raise ValueError(f"unknown SAM image encoder {name!r}: expected one of {sorted(VIT_CONFIGS)}")
    cfg = VIT_CONFIGS[name]
    return ImageEncoderViT(depth=cfg["depth"], embed_dim=cfg["embed_dim"], img_size=1024, mlp_ratio=4,
                           norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), num_heads=cfg["num_heads"], patch_size=16, qkv_bias=True,
                           use_rel_pos=True, global_attn_indexes=cfg["global_attn_indexes"], window_size=14, out_chans=256,
                           precision=precision)
