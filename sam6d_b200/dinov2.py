"""ISM descriptor branch on H100 kernels (SURVEY.md 8f row N2): drop-ins for
    DinoVisionTransformer (ViT-S/B/L/g 14 = dinov2_vit{s,b,l,g}14)   ISM/model/vision_transformer.py:43-392
    CustomDINOv2                                        ISM/model/dinov2.py:92-258
    MaskedPatch_MatrixSimilarity (compute_straight / compute_visible_ratio)   ISM/model/loss.py:46-77
    compute_appearance_score / compute_geometric_score  ISM/model/detector.py:298-323

The trunk is a pre-norm ViT with LayerScale: parameter names are the reference's (`cls_token`, `pos_embed` (1, 1370, C),
`mask_token`, `patch_embed.proj`, `blocks.N.{norm1, attn.{qkv,proj}, ls1.gamma, norm2, mlp.{fc1,fc2} or mlp.{w12,w3}, ls2.gamma}`, `norm`), so
`dinov2_vit{s,b,l,g}14_pretrain.pth` load unchanged.  Every forward runs through the C ABI:
    patch embedding, qkv / proj / fc1 / fc2                -> sam6d_gemm_tma / sam6d_gemm_tc (wgmma; bias, GELU, residual epilogues;
                                                              LayerScale folded into proj / fc2 when the weights are packed)
    ViT-g's SwiGLU FFN w12 / w3                            -> sam6d_gemm_tma act=3 (silu(gate) * up formed in the epilogue registers,
                                                              w12 rows interleaved in blocks of 128 when packed) / residual epilogue
    LayerNorm                                              -> sam6d_layernorm_bf16
    attention over 257 tokens (C / 64 heads x 64)          -> sam6d_attn_tc_ex on keys 0..255 (tensor cores, log-sum-exp out)
                                                              + sam6d_attn_merge_key for the 257th token
    crop / mask / nearest resize / pad of all proposals    -> sam6d_crop_resize_pad
    masked, normalised patch tokens                        -> sam6d_masked_patch_normalize
    appearance score + visible ratio                       -> sam6d_gemm_tma_batched (256 x 256 x C per proposal) + sam6d_appearance_reduce
There is no CPU path.  The positional-embedding interpolation (bicubic, once per input size) is weight preprocessing in torch."""
import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, ops
from .layers import _W, _f32, _Packed, _PatchEmbed, _Attention, _Mlp, block, pack_block, patch_embed, patch_rows


class _SwiGLUFFNFused(nn.Module):
    """SwiGLUFFNFused (ISM/model/layers/swiglu_ffn.py:45-63): w12 = [gate; up] rows, hidden = (int(hidden * 2 / 3) + 7) // 8 * 8"""

    def __init__(self, dim, hidden):
        super().__init__()
        hidden = (int(hidden * 2 / 3) + 7) // 8 * 8
        self.w12 = nn.Linear(dim, 2 * hidden)
        self.w3 = nn.Linear(hidden, dim)


FFN_LAYERS = {"mlp": _Mlp, "swiglufused": _SwiGLUFFNFused}


class _LayerScale(nn.Module):
    def __init__(self, dim, init_values):
        super().__init__()
        self.gamma = nn.Parameter(init_values * torch.ones(dim))


class _Block(nn.Module):
    def __init__(self, dim, mlp_ratio, init_values, ffn_layer="mlp"):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = _Attention(dim)
        self.ls1 = _LayerScale(dim, init_values)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = FFN_LAYERS[ffn_layer](dim, int(dim * mlp_ratio))
        self.ls2 = _LayerScale(dim, init_values)


class DinoVisionTransformer(nn.Module):
    """forward(x (B,3,H,W), is_training=False) -> x_norm_clstoken (B,C), or with is_training=True the reference's dict with
    'x_norm_clstoken' and 'x_norm_patchtokens' (vision_transformer.py:232-267, 325-330).  H, W multiples of the patch size with at
    most 256 patches (the 224 x 224 proposal crops of SAM-6D give 16 x 16)."""

    def __init__(self, img_size=518, patch_size=14, in_chans=3, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4.0, init_values=1.0,
                 interpolate_offset=0.1, interpolate_antialias=False, num_register_tokens=0, ffn_layer="mlp"):
        super().__init__()
        if embed_dim // num_heads != 64 or num_register_tokens or interpolate_antialias:
            raise ValueError("sam6d_b200 DinoVisionTransformer: head dim 64, no register tokens (dinov2_vit{s,b,l,g}14)")
        if ffn_layer not in FFN_LAYERS:
            raise NotImplementedError(f"sam6d_b200 DinoVisionTransformer: ffn_layer {ffn_layer!r} (supported: {', '.join(FFN_LAYERS)})")
        self.embed_dim, self.num_heads, self.patch_size, self.depth = embed_dim, num_heads, patch_size, depth
        self.ffn_layer = ffn_layer
        self.interpolate_offset = interpolate_offset
        self.patch_embed = _PatchEmbed(patch_size, in_chans, embed_dim)
        n = (img_size // patch_size) ** 2
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, n + 1, embed_dim))
        self.mask_token = nn.Parameter(torch.zeros(1, embed_dim))
        self.blocks = nn.ModuleList([_Block(embed_dim, mlp_ratio, init_values, ffn_layer) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim, eps=1e-6)
        self._packed = _Packed()
        self._pos_cache = {}

    # ---- weights in kernel form ------------------------------------------------------------------------------------
    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        C, P = self.embed_dim, self.patch_size
        K = 3 * P * P
        Kp = (K + 7) // 8 * 8                                 # 588 -> 592: the GEMM wants K % 8 == 0 (zero columns)
        pw = torch.zeros(C, Kp, dtype=torch.float32, device=self.cls_token.device)
        pw[:, :K] = _f32(self.patch_embed.proj.weight).reshape(C, K)
        w = dict(pe_w=_W(pw), pe_b=_f32(self.patch_embed.proj.bias), Kp=Kp, nw=_f32(self.norm.weight), nb=_f32(self.norm.bias),
                 blocks=[])
        for blk in self.blocks:
            g1, g2 = _f32(blk.ls1.gamma).double(), _f32(blk.ls2.gamma).double()
            # x + gamma * (W y + b) = x + (diag(gamma) W) y + gamma * b : LayerScale folded into the projection
            # Mlp: l1 / l2 = fc1 / fc2.  SwiGLU: l1 = w12 with its gate and up rows interleaved for gemm_tma(act=3), l2 = w3
            if self.ffn_layer == "swiglufused":
                f1w, f1b = ops.pack_swiglu_rows(_f32(blk.mlp.w12.weight)), ops.pack_swiglu_rows(_f32(blk.mlp.w12.bias))
                f2w, f2b = blk.mlp.w3.weight, blk.mlp.w3.bias
            else:
                f1w, f1b = blk.mlp.fc1.weight, blk.mlp.fc1.bias
                f2w, f2b = blk.mlp.fc2.weight, blk.mlp.fc2.bias
            w["blocks"].append(pack_block(
                blk.norm1, blk.attn.qkv.weight, blk.attn.qkv.bias,
                (_f32(blk.attn.proj.weight).double() * g1[:, None]).float(), (_f32(blk.attn.proj.bias).double() * g1).float(),
                blk.norm2, f1w, f1b, (_f32(f2w).double() * g2[:, None]).float(), (_f32(f2b).double() * g2).float()))
        return w

    def _pos(self, npatch, w, h):
        """interpolate_pos_encoding (vision_transformer.py:179-207) -> (cls row (C,), patch rows (npatch, C)) with cls_token added"""
        ck = (npatch, w, h, self._packed.key)
        if ck not in self._pos_cache:
            pe = self.pos_embed.detach().float()
            N = pe.shape[1] - 1
            if not (npatch == N and w == h):
                dim = pe.shape[-1]
                w0, h0 = w // self.patch_size + self.interpolate_offset, h // self.patch_size + self.interpolate_offset
                sq = math.sqrt(N)
                patch_pe = F.interpolate(pe[:, 1:].reshape(1, int(sq), int(sq), dim).permute(0, 3, 1, 2), scale_factor=(float(w0) / sq, float(h0) / sq),
                                         mode="bicubic", antialias=False)
                pe = torch.cat((pe[:, :1], patch_pe.permute(0, 2, 3, 1).reshape(1, -1, dim)), dim=1)
            cls = (self.cls_token.detach().float().reshape(-1) + pe[0, 0]).contiguous()
            self._pos_cache = {ck: (cls, pe[0, 1:].contiguous())}
        return self._pos_cache[ck]

    def _attention(self, qk, vt, B, S, C):
        H, d = self.num_heads, C // self.num_heads
        scale = d ** -0.5
        if S <= 256:
            return ops.attn_tc(qk, 0, qk, C, vt, B, H, S, S, d, scale, out_dtype=torch.bfloat16)
        # 257 tokens: keys 0..255 (class token + 255 patches) on the tensor cores, then the last patch token merged by log-sum-exp.
        # (The window starts at key 0 because a TMA box must start on a 16-byte boundary of the V^T rows.)
        out, lse = ops.attn_tc_ex(qk, 0, qk, C, vt, B, H, S, S - 1, d, scale, k_brows=S, k_row0=0, v_col0=0, want_lse=True)
        ops.attn_merge_key(qk, 0, qk, C, S, S - 1, vt, S - 1, lse, B, H, S, scale, out)
        return out

    @torch.no_grad()
    def forward_features(self, x, masks=None):
        if masks is not None:
            raise NotImplementedError("mask tokens are a training feature of DINOv2")
        if not x.is_cuda:
            raise RuntimeError("sam6d_b200 DinoVisionTransformer needs CUDA tensors: there is no CPU path")
        w = self._weights()
        B, Cin, Himg, Wimg = x.shape
        P, C = self.patch_size, self.embed_dim
        Gh, Gw = Himg // P, Wimg // P
        L, S = Gh * Gw, Gh * Gw + 1
        if Himg % P or Wimg % P or L > 256:
            raise RuntimeError("input must be a multiple of the patch size with at most 256 patches")
        cls, pos = self._pos(L, Himg, Wimg)
        rows = patch_rows(x, P, w["Kp"])
        tok = torch.empty(B, S, C, dtype=torch.float32, device=x.device)
        tok[:, 0, :] = cls
        patch_embed("bf16", rows, w["pe_w"], w["pe_b"], pos, tok[:, 1:, :])
        tok = tok.view(B * S, C)
        act = ops.ACT_SWIGLU if self.ffn_layer == "swiglufused" else ops.ACT_GELU
        for bw in w["blocks"]:
            def attend(xn):
                qk, vt = ops.gemm_tma_vt(xn, bw["qkv"].bf16, bw["qkv_b"], 2 * C, S, slot=4)
                return self._attention(qk, vt, B, S, C)
            tok = block("bf16", bw, tok, attend, act)
        xn = ops.layernorm(tok, w["nw"], w["nb"], eps=1e-6).view(B, S, C)
        return {"x_norm_clstoken": xn[:, 0], "x_norm_regtokens": xn[:, 1:1], "x_norm_patchtokens": xn[:, 1:], "x_prenorm": tok.view(B, S, C),
                "masks": masks}

    @torch.no_grad()
    def forward(self, *args, is_training=False, **kwargs):
        ret = self.forward_features(*args, **kwargs)
        return ret if is_training else ret["x_norm_clstoken"]


def _vit(patch_size, embed_dim, depth, num_heads, kwargs):
    """the constructors of vision_transformer.py:336-392 with the arguments of _make_dinov2_model (dinov2.py:46-90)"""
    kw = dict(img_size=518, init_values=1.0, embed_dim=embed_dim, depth=depth, num_heads=num_heads, mlp_ratio=4)
    kw.update(kwargs)
    return DinoVisionTransformer(patch_size=patch_size, **kw)


def vit_small(patch_size=14, **kwargs):
    """dinov2_vits14 (vision_transformer.py:336-347)"""
    return _vit(patch_size, 384, 12, 6, kwargs)


def vit_base(patch_size=14, **kwargs):
    """dinov2_vitb14 (vision_transformer.py:350-361)"""
    return _vit(patch_size, 768, 12, 12, kwargs)


def vit_large(patch_size=14, **kwargs):
    """dinov2_vitl14 (vision_transformer.py:364-375 with the arguments of _make_dinov2_model, dinov2.py:46-90)"""
    return _vit(patch_size, 1024, 24, 16, kwargs)


def vit_giant2(patch_size=14, **kwargs):
    """vision_transformer.py:378-392 (1536 / 24 heads of 64 / 40 blocks); dinov2_vitg14 passes ffn_layer='swiglufused'"""
    return _vit(patch_size, 1536, 40, 24, kwargs)


# ISM/model/dinov2.py:14-26
descriptor_size = {"dinov2_vits14": 384, "dinov2_vitb14": 768, "dinov2_vitl14": 1024, "dinov2_vitg14": 1536}
descriptor_map = {"dinov2_vits14": "vit_small", "dinov2_vitb14": "vit_base", "dinov2_vitl14": "vit_large", "dinov2_vitg14": "vit_giant2"}
_CONSTRUCTORS = {"vit_small": vit_small, "vit_base": vit_base, "vit_large": vit_large, "vit_giant2": vit_giant2}
# The reference builds every backbone with the default Mlp FFN, but the published dinov2_vitg14_pretrain.pth holds SwiGLU weights
# (blocks.N.mlp.w12 / w3), which its strict load_state_dict rejects.  Here ViT-g is built as the checkpoint is: SwiGLUFFNFused.
FFN_OF_MODEL = {"dinov2_vitg14": "swiglufused"}


def build_descriptor_vit(model_name, patch_size=14):
    """the backbone of CustomDINOv2(model_name): dinov2_vit{s,b,l,g}14 -> DinoVisionTransformer"""
    if model_name not in descriptor_map:
        raise NotImplementedError(f"DINOv2 model {model_name!r}: sam6d_b200 supports {', '.join(descriptor_map)} (no register-token variants)")
    return _CONSTRUCTORS[descriptor_map[model_name]](patch_size, ffn_layer=FFN_OF_MODEL.get(model_name, "mlp"))


# =====================================================================================================================
def crop_resize_pad(image_u8: Optional[torch.Tensor], masks: torch.Tensor, boxes: torch.Tensor, target: int = 224, want_rgb=True, want_mask=True):
    """all proposals of a frame in one launch pair: image (H,W,3) uint8, masks (P,H,W) float, boxes (P,4) xyxy
    -> (rgb (P,3,T,T) or None, mask (P,T,T) or None)   (CustomDINOv2.process_rgb_proposals / process_masks_proposals)"""
    P, H, W = masks.shape
    dev = masks.device
    m = masks.float().contiguous()
    b = boxes.to(torch.int32).contiguous()
    rgb = torch.empty(P, 3, target, target, dtype=torch.float32, device=dev) if want_rgb else None
    pm = torch.empty(P, target, target, dtype=torch.float32, device=dev) if want_mask else None
    img = image_u8.contiguous() if want_rgb else None
    _lib.call("sam6d_crop_resize_pad", img, m, b, P, H, W, target, rgb, pm)
    return rgb, pm


class CustomDINOv2(nn.Module):
    """ISM/model/dinov2.py:92-258 without the Lightning base: forward(image_np (H,W,3) uint8, proposals with .masks (P,H,W) and
    .boxes (P,4)) -> (cls_features (P,C), patch_features (P,256,C) masked + L2-normalised)."""

    def __init__(self, model_name="dinov2_vitl14", token_name="x_norm_clstoken", image_size=224, chunk_size=16, descriptor_width_size=640,
                 checkpoint_dir=None, patch_size=14, validpatch_thresh=0.5, model: Optional[nn.Module] = None):
        super().__init__()
        self.model_name = model_name
        self.model = model if model is not None else build_descriptor_vit(model_name, patch_size)
        if checkpoint_dir is not None:
            import os.path as osp
            self.model.load_state_dict(torch.load(osp.join(checkpoint_dir, f"{model_name}_pretrain.pth"), map_location="cpu"))
        self.validpatch_thresh, self.token_name, self.chunk_size = validpatch_thresh, token_name, chunk_size
        self.patch_size, self.proposal_size, self.descriptor_width_size = patch_size, image_size, descriptor_width_size

    def _image(self, image_np, device):
        img = image_np if torch.is_tensor(image_np) else torch.from_numpy(image_np)
        return img.to(device=device, dtype=torch.uint8).contiguous()

    @torch.no_grad()
    def process_rgb_proposals(self, image_np, masks, boxes):
        return crop_resize_pad(self._image(image_np, masks.device), masks, boxes, self.proposal_size, True, False)[0]

    @torch.no_grad()
    def process_masks_proposals(self, masks, boxes):
        return crop_resize_pad(None, masks, boxes, self.proposal_size, False, True)[1]

    @torch.no_grad()
    def compute_cls_and_patch_features(self, images, masks, want_bf16=False):
        """dinov2.py:248-258 (+ the bf16 copy / validity flags the scoring kernels use)"""
        P = images.shape[0]
        C, G = self.model.embed_dim, self.proposal_size // self.patch_size
        cls = torch.empty(P, C, dtype=torch.float32, device=images.device)
        pf = torch.empty(P, G * G, C, dtype=torch.float32, device=images.device)
        pb = torch.empty(P, G * G, C, dtype=torch.bfloat16, device=images.device) if want_bf16 else None
        valid = torch.empty(P, G * G, dtype=torch.uint8, device=images.device)
        chunk = max(self.chunk_size, 64)          # the reference's 16 bounds eager-attention memory; the kernels batch more
        for i in range(0, P, chunk):
            f = self.model(images[i:i + chunk].contiguous(), is_training=True)
            n = f["x_norm_clstoken"].shape[0]
            cls[i:i + n] = f["x_norm_clstoken"]
            pt = f["x_norm_patchtokens"]                                     # view of (n, S, C): row stride C, batch stride S*C
            mk = masks[i:i + n].contiguous()                                 # named: must outlive the launch
            _lib.call("sam6d_masked_patch_normalize", pt, pt.stride(1), pt.stride(0), mk, n, G, self.patch_size, C, self.validpatch_thresh,
                      pf[i:i + n], pb[i:i + n] if want_bf16 else None, valid[i:i + n])
        self.last_patch_bf16, self.last_valid = pb, valid
        return cls, pf

    @torch.no_grad()
    def forward(self, image_np, proposals, want_bf16=False):
        masks, boxes = proposals.masks, proposals.boxes
        rgbs, pmasks = crop_resize_pad(self._image(image_np, masks.device), masks, boxes, self.proposal_size, True, True)
        return self.compute_cls_and_patch_features(rgbs, pmasks, want_bf16)

    @torch.no_grad()
    def forward_cls_token(self, image_np, proposals):
        return self.forward(image_np, proposals)[0]

    @torch.no_grad()
    def forward_patch_tokens(self, image_np, proposals):
        return self.forward(image_np, proposals)[1]


class MaskedPatch_MatrixSimilarity(nn.Module):
    """ISM/model/loss.py:46-77: compute_straight (appearance score) and compute_visible_ratio on (P, N, C) patch descriptors
    (masked rows are zero), N <= 256.  One batched tensor-core GEMM + one reduction kernel produce both."""

    def __init__(self, metric="cosine", chunk_size=64):
        super().__init__()
        self.metric, self.chunk_size = metric, chunk_size

    @torch.no_grad()
    def scores(self, query, reference, thred=0.5):
        P, N, C = query.shape
        q = query.to(torch.bfloat16).contiguous()
        r = reference.to(torch.bfloat16).contiguous()
        ld = (N + 3) // 4 * 4
        sim = torch.empty(P, N, ld, dtype=torch.float32, device=query.device)
        ops.gemm_tma_batched(q, r, sim[:, :, :N])
        qvalid = (query.abs().amax(dim=-1) > 0).to(torch.uint8).contiguous()
        appe = torch.empty(P, dtype=torch.float32, device=query.device)
        vis = torch.empty(P, dtype=torch.float32, device=query.device)
        _lib.call("sam6d_appearance_reduce", sim, ld, N * ld, P, N, qvalid, thred, appe, vis)
        return appe, vis

    def compute_straight(self, query, reference):
        return self.scores(query, reference)[0]

    def compute_visible_ratio(self, query, reference, thred=0.5):
        return self.scores(query, reference, thred)[1]


def compute_appearance_score(ref_appe_descriptors_all, best_pose, pred_objects_idx, query_appe_descriptors):
    """detector.py:298-309: gather the best template's patch descriptors per proposal, then compute_straight"""
    ref = ref_appe_descriptors_all[pred_objects_idx, best_pose, ...]
    return MaskedPatch_MatrixSimilarity().compute_straight(query_appe_descriptors, ref), ref
