"""SAM prompt encoder, mask decoder, predictor and automatic mask generator on H100 kernels (SURVEY.md 8f row N4): drop-ins for
    PromptEncoder (points, boxes, masks) ISM/segment_anything/modeling/prompt_encoder.py:16-214
    MaskDecoder / TwoWayTransformer      ISM/segment_anything/modeling/{mask_decoder,transformer}.py
    Sam (preprocess / postprocess)       ISM/segment_anything/modeling/sam.py
    SamPredictor / ResizeLongestSide     ISM/segment_anything/{predictor.py,utils/transforms.py}; load_sam_predictor ISM/model/sam.py:32-39
    CustomSamAutomaticMaskGenerator      ISM/model/sam.py:52-155 over SamAutomaticMaskGenerator (automatic_mask_generator.py)
with the reference's module and parameter names (`sam_vit_{h,l,b}_*.pth` load unchanged: `image_encoder.*`, `prompt_encoder.*`,
`mask_decoder.*`).  `sam_model_registry` and `load_sam` are the reference's entry points for picking the backbone (vit_h, vit_l,
vit_b); the prompt encoder and mask decoder are the same for all three.

Work split.  Every Linear of the decoder -- token side and image side, and the two transposed convolutions written as GEMMs over
pixel rows -- runs on the wgmma GEMMs (`sam6d_gemm_tma(_batched)` for the 262 144-row image side of a 64-prompt batch,
`sam6d_gemm_f32` for the 448-row token side); csrc/sam_dec.cu holds the mask-prompt embedding, the attention cores (up to 32 tokens <-> 4096 pixels, head
dims 16 / 32), LayerNorm2d + GELU, the hypernetwork product with both pixel shuffles folded into its output index, and the mask
post-processing.  Three algebraic savings over the reference's formulation, all exact:
  * in block 0 the image-side keys are the same for all 64 prompts (src + no-mask embedding): their k / v / q projections are
    computed once per FRAME, not once per prompt (prompts with a mask input have their own src + dense and their own projections);
  * `proj(keys + pe) = proj(keys) + W pe`: the positional term of every image-side projection is one (4096 x 128) matrix per frame,
    added as a shared residual in the GEMM epilogue instead of a (64, 4096, 256) elementwise pass;
  * `Sam.postprocess_masks` (256 -> 1024 bilinear, crop, -> frame size bilinear) is evaluated per output pixel inside the statistics
    kernel: the (64, 3, 1024, 1024) and (64, 3, H, W) logit tensors never exist; only kept masks are materialised (binary).
The reference's RLE encode / decode round trip inside `_generate_masks` is the identity and is skipped."""
import math
import os
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops
from .layers import _W, _f32, _Packed
from .sam import LayerNorm2d

bf = torch.bfloat16


class _PositionEmbeddingRandom(nn.Module):
    def __init__(self, num_pos_feats=128):
        super().__init__()
        self.register_buffer("positional_encoding_gaussian_matrix", torch.randn(2, num_pos_feats))


def _pe_encode(coords01: torch.Tensor, G: torch.Tensor) -> torch.Tensor:
    """coords (rows,2) in [0,1] -> (rows,256)"""
    c = coords01.float().contiguous()
    g = G.float().contiguous()                           # named: must outlive the launch
    out = torch.empty(c.shape[0], 256, dtype=torch.float32, device=c.device)
    _lib.call("sam6d_sam_pe_encode", c, g, c.shape[0], out)
    return out


MAX_PROMPT_TOKENS = 27          # sparse tokens per prompt the decoder kernels take: 5 output tokens + 27 <= 32


class PromptEncoder(nn.Module):
    """point, box and mask prompts (prompt_encoder.py:16-214): sparse embeddings in the reference's order (points, padding point
    when there is no box, box corners); the dense embedding of a mask prompt comes from `sam6d_sam_mask_embed` as token rows"""

    def __init__(self, embed_dim=256, image_embedding_size=(64, 64), input_image_size=(1024, 1024), mask_in_chans=16, activation=nn.GELU):
        super().__init__()
        self.embed_dim, self.input_image_size, self.image_embedding_size = embed_dim, input_image_size, image_embedding_size
        self.pe_layer = _PositionEmbeddingRandom(embed_dim // 2)
        self.num_point_embeddings = 4
        self.point_embeddings = nn.ModuleList([nn.Embedding(1, embed_dim) for _ in range(4)])
        self.not_a_point_embed = nn.Embedding(1, embed_dim)
        self.mask_input_size = (4 * image_embedding_size[0], 4 * image_embedding_size[1])
        self.mask_downscaling = nn.Sequential(
            nn.Conv2d(1, mask_in_chans // 4, kernel_size=2, stride=2), LayerNorm2d(mask_in_chans // 4), activation(),
            nn.Conv2d(mask_in_chans // 4, mask_in_chans, kernel_size=2, stride=2), LayerNorm2d(mask_in_chans), activation(),
            nn.Conv2d(mask_in_chans, embed_dim, kernel_size=1))
        self.no_mask_embed = nn.Embedding(1, embed_dim)
        self._packed = _Packed()

    @torch.no_grad()
    def dense_pe_rows(self) -> torch.Tensor:
        """get_dense_pe as token rows: (h*w, 256), row = y*w + x"""
        h, w = self.image_embedding_size
        dev = self.no_mask_embed.weight.device
        ys, xs = torch.meshgrid((torch.arange(h, device=dev) + 0.5) / h, (torch.arange(w, device=dev) + 0.5) / w, indexing="ij")
        return _pe_encode(torch.stack([xs, ys], dim=-1).reshape(-1, 2), self.pe_layer.positional_encoding_gaussian_matrix)

    @torch.no_grad()
    def get_dense_pe(self) -> torch.Tensor:
        h, w = self.image_embedding_size
        return self.dense_pe_rows().view(h, w, -1).permute(2, 0, 1).unsqueeze(0)

    def _mask_params(self) -> torch.Tensor:
        """mask_downscaling's parameters in the order sam6d_sam_mask_embed reads them (include/sam6d_b200.h)"""
        md = self.mask_downscaling
        params = (md[0].weight, md[0].bias, md[1].weight, md[1].bias, md[3].weight, md[3].bias, md[4].weight, md[4].bias, md[6].weight, md[6].bias)
        return self._packed.get(lambda: torch.cat([_f32(t).reshape(-1) for t in params]).contiguous(), md)

    def _pe(self, coords: torch.Tensor) -> torch.Tensor:
        """PositionEmbeddingRandom.forward_with_coords: (B,N,2) pixel coordinates, already shifted by 0.5 -> (B,N,256)"""
        B, N, _ = coords.shape
        c = torch.stack([coords[..., 0] / self.input_image_size[1], coords[..., 1] / self.input_image_size[0]], dim=-1)
        return _pe_encode(c.reshape(-1, 2), self.pe_layer.positional_encoding_gaussian_matrix).view(B, N, -1)

    @torch.no_grad()
    def embed_masks(self, masks: torch.Tensor) -> torch.Tensor:
        """mask_downscaling of (B,1,256,256) logits -> (B,256,64,64), a view of the (B,4096,256) token rows the decoder reads"""
        B = masks.shape[0]
        h, w = self.image_embedding_size
        if masks.dim() != 4 or tuple(masks.shape[1:]) != (1, 4 * h, 4 * w) or (h, w) != (64, 64) or self.embed_dim != 256:
            raise ValueError(f"mask prompts must be (B, 1, 256, 256) low-res logits, got {tuple(masks.shape)}")
        m = masks.to(device=self.no_mask_embed.weight.device, dtype=torch.float32).contiguous()
        prm = self._mask_params()
        rows = torch.empty(B, h * w, self.embed_dim, dtype=torch.float32, device=m.device)
        _lib.call("sam6d_sam_mask_embed", m, prm, B, rows)
        return rows.view(B, h, w, self.embed_dim).permute(0, 3, 1, 2)

    @torch.no_grad()
    def forward(self, points, boxes=None, masks=None):
        bs = points[0].shape[0] if points is not None else boxes.shape[0] if boxes is not None else masks.shape[0] if masks is not None else 1
        for name, t in (("point labels", points[1] if points is not None else None), ("boxes", boxes), ("masks", masks)):
            if t is not None and t.shape[0] != bs:
                raise ValueError(f"prompt batch sizes differ: {name} has {t.shape[0]}, expected {bs}")
        if masks is not None and (masks.dim() != 4 or tuple(masks.shape[1:]) != (1,) + tuple(self.mask_input_size)):
            raise ValueError(f"mask_input must be (B, 1, {self.mask_input_size[0]}, {self.mask_input_size[1]}), got {tuple(masks.shape)}")
        n_sparse = (points[0].shape[1] + (boxes is None) if points is not None else 0) + (2 if boxes is not None else 0)
        if n_sparse > MAX_PROMPT_TOKENS:
            raise ValueError(f"{n_sparse} prompt tokens per prompt: the decoder takes at most {MAX_PROMPT_TOKENS} "
                             "(26 points and the padding point, or 25 points and a box)")
        dev = self.no_mask_embed.weight.device
        parts = []
        if points is not None:
            coords, labels = points
            B, N, _ = coords.shape
            e = self._pe(coords.to(dev).float() + 0.5)
            lab = labels.to(dev).reshape(B, N)
            zero = torch.zeros_like(e)
            e = torch.where((lab == -1)[..., None], zero, e)                                   # _embed_points: PE of a -1 point zeroed
            e = e + torch.where((lab == 1)[..., None], self.point_embeddings[1].weight, zero) + \
                torch.where((lab == 0)[..., None], self.point_embeddings[0].weight, zero) + \
                torch.where((lab == -1)[..., None], self.not_a_point_embed.weight, zero)
            parts.append(e)
            if boxes is None:
                parts.append(self.not_a_point_embed.weight.view(1, 1, -1).expand(B, 1, -1))      # padding point: PE zeroed, label -1
        if boxes is not None:
            c = self._pe(boxes.to(dev).float().reshape(-1, 2, 2) + 0.5)                         # _embed_boxes
            parts.append(c + torch.cat([self.point_embeddings[2].weight, self.point_embeddings[3].weight], dim=0))
        sparse = torch.cat(parts, dim=1).contiguous() if parts else torch.empty(bs, 0, self.embed_dim, device=dev)
        h, w = self.image_embedding_size
        if masks is not None:
            dense = self.embed_masks(masks)
        else:
            dense = self.no_mask_embed.weight.reshape(1, -1, 1, 1).expand(bs, -1, h, w)
        return sparse, dense


class _Attention(nn.Module):
    def __init__(self, dim, heads, downsample_rate=1):
        super().__init__()
        self.internal_dim, self.num_heads = dim // downsample_rate, heads
        self.q_proj, self.k_proj, self.v_proj = nn.Linear(dim, self.internal_dim), nn.Linear(dim, self.internal_dim), nn.Linear(dim, self.internal_dim)
        self.out_proj = nn.Linear(self.internal_dim, dim)


class _MLPBlock(nn.Module):
    def __init__(self, dim, mlp_dim):
        super().__init__()
        self.lin1, self.lin2 = nn.Linear(dim, mlp_dim), nn.Linear(mlp_dim, dim)


class _TwoWayAttentionBlock(nn.Module):
    def __init__(self, dim, heads, mlp_dim, downsample, skip_first_layer_pe):
        super().__init__()
        self.self_attn = _Attention(dim, heads)
        self.norm1 = nn.LayerNorm(dim)
        self.cross_attn_token_to_image = _Attention(dim, heads, downsample)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = _MLPBlock(dim, mlp_dim)
        self.norm3 = nn.LayerNorm(dim)
        self.norm4 = nn.LayerNorm(dim)
        self.cross_attn_image_to_token = _Attention(dim, heads, downsample)
        self.skip_first_layer_pe = skip_first_layer_pe


class TwoWayTransformer(nn.Module):
    def __init__(self, depth=2, embedding_dim=256, num_heads=8, mlp_dim=2048, activation=nn.ReLU, attention_downsample_rate=2):
        super().__init__()
        if (depth, embedding_dim, num_heads, attention_downsample_rate) != (2, 256, 8, 2):
            raise ValueError("sam6d_b200 TwoWayTransformer is built for SAM's configuration (depth 2, dim 256, 8 heads, downsample 2)")
        self.layers = nn.ModuleList([_TwoWayAttentionBlock(embedding_dim, num_heads, mlp_dim, attention_downsample_rate, i == 0) for i in range(depth)])
        self.final_attn_token_to_image = _Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.norm_final_attn = nn.LayerNorm(embedding_dim)


class _MLP(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        h = [hidden_dim] * (num_layers - 1)
        self.num_layers = num_layers
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))


def _lin(x2d, lin: nn.Linear, relu=False, residual=None):
    """token-side Linear on the fp32 CUDA-core GEMM (a few hundred rows)"""
    return ops.gemm(x2d.contiguous(), _f32(lin.weight), _f32(lin.bias), residual=residual, relu=relu)


def _ln(x2d, ln: nn.LayerNorm):
    return ops.layernorm(x2d.contiguous(), _f32(ln.weight), _f32(ln.bias), eps=ln.eps)


class MaskDecoder(nn.Module):
    def __init__(self, *, transformer_dim=256, transformer: Optional[nn.Module] = None, num_multimask_outputs=3, activation=nn.GELU,
                 iou_head_depth=3, iou_head_hidden_dim=256):
        super().__init__()
        self.transformer_dim = transformer_dim
        self.transformer = transformer if transformer is not None else TwoWayTransformer()
        self.num_multimask_outputs = num_multimask_outputs
        self.iou_token = nn.Embedding(1, transformer_dim)
        self.num_mask_tokens = num_multimask_outputs + 1
        self.mask_tokens = nn.Embedding(self.num_mask_tokens, transformer_dim)
        self.output_upscaling = nn.Sequential(
            nn.ConvTranspose2d(transformer_dim, transformer_dim // 4, kernel_size=2, stride=2), LayerNorm2d(transformer_dim // 4), activation(),
            nn.ConvTranspose2d(transformer_dim // 4, transformer_dim // 8, kernel_size=2, stride=2), activation())
        self.output_hypernetworks_mlps = nn.ModuleList([_MLP(transformer_dim, transformer_dim, transformer_dim // 8, 3) for _ in range(self.num_mask_tokens)])
        self.iou_prediction_head = _MLP(transformer_dim, iou_head_hidden_dim, self.num_mask_tokens, iou_head_depth)
        self._packed = _Packed()
        self._frame = {}

    # ---- weights in kernel form -----------------------------------------------------------------------------------------------
    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        t = self.transformer
        w = {}
        for name, a in (("t2i0", t.layers[0].cross_attn_token_to_image), ("i2t0", t.layers[0].cross_attn_image_to_token),
                        ("t2i1", t.layers[1].cross_attn_token_to_image), ("i2t1", t.layers[1].cross_attn_image_to_token),
                        ("fin", t.final_attn_token_to_image)):
            w[name] = dict(q=_W(a.q_proj.weight), qb=_f32(a.q_proj.bias), k=_W(a.k_proj.weight), kb=_f32(a.k_proj.bias),
                           v=_W(a.v_proj.weight), vb=_f32(a.v_proj.bias), o=_W(a.out_proj.weight), ob=_f32(a.out_proj.bias))
        up = self.output_upscaling
        w["ct1"] = _W(_f32(up[0].weight).permute(2, 3, 1, 0).reshape(4 * up[0].out_channels, up[0].in_channels))     # rows (i, j, o)
        w["ct1b"] = _f32(up[0].bias).repeat(4).contiguous()
        w["ln2w"], w["ln2b"] = _f32(up[1].weight), _f32(up[1].bias)
        w["ct2"] = _W(_f32(up[3].weight).permute(2, 3, 1, 0).reshape(4 * up[3].out_channels, up[3].in_channels))
        w["ct2b"] = _f32(up[3].bias).repeat(4).contiguous()
        return w

    def _frame_terms(self, image_embeddings, pe_rows, no_mask):
        """everything that depends on the frame but not on the prompts (block 0 of the transformer sees the same image tokens for
        every prompt) -- computed once per image embedding"""
        fk = (image_embeddings.data_ptr(), image_embeddings._version, self._packed.key)
        if self._frame.get("key") != fk:
            w = self._weights()
            L = image_embeddings.shape[-2] * image_embeddings.shape[-1]
            src0 = (image_embeddings[0].reshape(256, L).t() + no_mask.reshape(1, 256)).contiguous()              # (L,256) f32
            src0_bf = src0.to(bf)
            srcpe_bf = (src0 + pe_rows).to(bf)
            f = dict(key=fk, src0_bf=src0_bf, L=L)
            a = w["t2i0"]
            f["K0"] = ops.gemm_tma(srcpe_bf, a["k"].bf16, a["kb"], out_dtype=bf)
            f["V0"] = ops.gemm_tma(src0_bf, a["v"].bf16, a["vb"], out_dtype=bf)
            f["Q0"] = ops.gemm_tma(srcpe_bf, w["i2t0"]["q"].bf16, w["i2t0"]["qb"], out_dtype=bf)
            f.update(self._pe_terms(pe_rows))
            self._frame = f
        return self._frame

    def _pe_terms(self, pe_rows):
        """W pe (no bias) of the image-side projections after block 0, added as shared residuals"""
        w = self._weights()
        pe_bf = pe_rows.to(bf).contiguous()
        return dict(peK1=ops.gemm_tma(pe_bf, w["t2i1"]["k"].bf16, None, out_dtype=bf),
                    peQ1=ops.gemm_tma(pe_bf, w["i2t1"]["q"].bf16, None, out_dtype=bf),
                    peKf=ops.gemm_tma(pe_bf, w["fin"]["k"].bf16, None, out_dtype=bf))

    def _prompt_terms(self, image_embeddings, pe_rows, dense):
        """block 0's image terms when every prompt has its own dense embedding (mask prompts): src_b = img + dense_b, and
        K0 / V0 / Q0 over all B*L rows, with per-prompt strides"""
        w = self._weights()
        B = dense.shape[0]
        L = image_embeddings.shape[-2] * image_embeddings.shape[-1]
        rows = dense.permute(0, 2, 3, 1).reshape(B, L, 256)                           # a view when dense came from embed_masks
        img = image_embeddings[0].reshape(256, L).t().float().contiguous()             # (L,256)
        src = torch.add(img, rows, out=torch.empty(B, L, 256, dtype=torch.float32, device=img.device))   # the reference's src + dense
        src_bf = src.to(bf).view(B * L, 256)
        srcpe_bf = (src + pe_rows).to(bf).view(B * L, 256)
        del src
        f = dict(L=L, src0_bf=src_bf, kv_bs=L * 128)
        a = w["t2i0"]
        f["K0"] = ops.gemm_tma(srcpe_bf, a["k"].bf16, a["kb"], out_dtype=bf)
        f["V0"] = ops.gemm_tma(src_bf, a["v"].bf16, a["vb"], out_dtype=bf)
        f["Q0"] = ops.gemm_tma(srcpe_bf, w["i2t0"]["q"].bf16, w["i2t0"]["qb"], out_dtype=bf)
        f.update(self._pe_terms(pe_rows))
        return f

    def _img_proj(self, keys_bf, W, b, pe_term, B, L):
        """proj(keys + pe) = keys W^T + b + (pe W^T): (B,L,256) bf16 -> (B,L,128) bf16, the pe term as a residual shared by all prompts"""
        out = torch.empty(B, L, 128, dtype=bf, device=keys_bf.device)
        return ops.gemm_tma_batched(keys_bf, W, out, bias=b, residual=pe_term.expand(B, L, 128))

    @staticmethod
    def _shared_dense(dense) -> bool:
        """the no-mask embedding broadcast over prompts and pixels (what PromptEncoder returns without a mask prompt)"""
        return dense.stride(2) == 0 and dense.stride(3) == 0 and (dense.shape[0] == 1 or dense.stride(0) == 0)

    @torch.no_grad()
    def predict_masks(self, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings, multimask_output=True):
        w = self._weights()
        t = self.transformer
        B, T = sparse_prompt_embeddings.shape[0], sparse_prompt_embeddings.shape[1] + self.num_mask_tokens + 1
        dev = sparse_prompt_embeddings.device
        if image_embeddings.shape[0] != 1:
            raise NotImplementedError("one image embedding per call (SamPredictor semantics)")
        if T > 5 + MAX_PROMPT_TOKENS:
            raise ValueError(f"{T - 5} prompt tokens per prompt: the decoder takes at most {MAX_PROMPT_TOKENS}")
        if dense_prompt_embeddings.shape[0] != B:
            raise ValueError(f"dense embeddings for {dense_prompt_embeddings.shape[0]} prompts, sparse for {B}")
        pe_rows = image_pe[0].reshape(256, -1).t().contiguous() if image_pe.dim() == 4 else image_pe
        if self._shared_dense(dense_prompt_embeddings):
            f = self._frame_terms(image_embeddings, pe_rows, dense_prompt_embeddings[0, :, 0, 0])
            kv_bs0 = 0
        else:
            f = self._prompt_terms(image_embeddings, pe_rows, dense_prompt_embeddings)
            kv_bs0 = f["kv_bs"]
        L = f["L"]
        out_tokens = torch.cat([self.iou_token.weight, self.mask_tokens.weight], dim=0)
        tokens = torch.cat((out_tokens.unsqueeze(0).expand(B, -1, -1), sparse_prompt_embeddings), dim=1).float().contiguous()   # (B,T,256)
        tok2 = tokens.view(B * T, 256)

        def self_attn(a, q_in, k_in, v_in):
            q, k, v = _lin(q_in, a.q_proj), _lin(k_in, a.k_proj), _lin(v_in, a.v_proj)
            o = torch.empty_like(q)
            _lib.call("sam6d_sam_self_attn", q, k, v, B, T, o)
            return o

        def tok2img(a, aw, q_in, K, V, kv_bs):
            q = _lin(q_in, a.q_proj)                                             # (B*T,128)
            o = torch.empty_like(q)
            _lib.call("sam6d_sam_tok2img_attn", q, K, V, kv_bs, B, T, L, o)
            return o

        def img2tok(a, Qimg, q_bs, k_in, v_in):
            kt, vt = _lin(k_in, a.k_proj), _lin(v_in, a.v_proj)                 # (B*T,128)
            o = torch.empty(B, L, 128, dtype=bf, device=dev)
            _lib.call("sam6d_sam_img2tok_attn", Qimg, q_bs, kt, vt, B, T, L, o)
            return o

        # ---- block 0 (skip_first_layer_pe) ----------------------------------------------------------------------------------
        l0, l1 = t.layers[0], t.layers[1]
        q = _ln(_lin(self_attn(l0.self_attn, tok2, tok2, tok2), l0.self_attn.out_proj), l0.norm1)
        a = tok2img(l0.cross_attn_token_to_image, w["t2i0"], q + tok2, f["K0"], f["V0"], kv_bs0)
        q = _ln(_lin(a, l0.cross_attn_token_to_image.out_proj, residual=q), l0.norm2)
        q = _ln(_lin(_lin(q, l0.mlp.lin1, relu=True), l0.mlp.lin2, residual=q), l0.norm3)
        a = img2tok(l0.cross_attn_image_to_token, f["Q0"], kv_bs0, q + tok2, q)
        keys = torch.empty(B, L, 256, dtype=bf, device=dev)
        ops.gemm_tma_batched(a, w["i2t0"]["o"].bf16, keys, bias=w["i2t0"]["ob"], residual=f["src0_bf"].view(-1, L, 256).expand(B, L, 256))
        keys = ops.layernorm_bf16io(keys.view(B * L, 256), _f32(l0.norm4.weight), _f32(l0.norm4.bias), eps=l0.norm4.eps).view(B, L, 256)
        # ---- block 1 -----------------------------------------------------------------------------------------------------------
        qp = q + tok2
        q = _ln(_lin(self_attn(l1.self_attn, qp, qp, q), l1.self_attn.out_proj, residual=q), l1.norm1)
        K1 = self._img_proj(keys, w["t2i1"]["k"].bf16, w["t2i1"]["kb"], f["peK1"], B, L)
        V1 = ops.gemm_tma(keys.view(B * L, 256), w["t2i1"]["v"].bf16, w["t2i1"]["vb"], out_dtype=bf)
        a = tok2img(l1.cross_attn_token_to_image, w["t2i1"], q + tok2, K1, V1, L * 128)
        q = _ln(_lin(a, l1.cross_attn_token_to_image.out_proj, residual=q), l1.norm2)
        q = _ln(_lin(_lin(q, l1.mlp.lin1, relu=True), l1.mlp.lin2, residual=q), l1.norm3)
        Q1 = self._img_proj(keys, w["i2t1"]["q"].bf16, w["i2t1"]["qb"], f["peQ1"], B, L)
        a = img2tok(l1.cross_attn_image_to_token, Q1, L * 128, q + tok2, q)
        k2 = ops.gemm_tma(a.view(B * L, 128), w["i2t1"]["o"].bf16, w["i2t1"]["ob"], residual=keys.view(B * L, 256), out_dtype=bf)
        keys = ops.layernorm_bf16io(k2, _f32(l1.norm4.weight), _f32(l1.norm4.bias), eps=l1.norm4.eps).view(B, L, 256)
        # ---- final token -> image attention ---------------------------------------------------------------------------------------
        Kf = self._img_proj(keys, w["fin"]["k"].bf16, w["fin"]["kb"], f["peKf"], B, L)
        Vf = ops.gemm_tma(keys.view(B * L, 256), w["fin"]["v"].bf16, w["fin"]["vb"], out_dtype=bf)
        a = tok2img(t.final_attn_token_to_image, w["fin"], q + tok2, Kf, Vf, L * 128)
        q = _ln(_lin(a, t.final_attn_token_to_image.out_proj, residual=q), t.norm_final_attn)
        hs = q.view(B, T, 256)
        # ---- upscaling: two transposed convolutions as GEMMs over pixel rows, hypernetwork product ---------------------------------
        G = int(math.isqrt(L))
        u1 = ops.gemm_tma(keys.view(B * L, 256), w["ct1"].bf16, w["ct1b"], out_dtype=bf)                   # (B*L, 4*64): cols (i,j,o)
        u1n = torch.empty_like(u1)
        _lib.call("sam6d_sam_ln2d_gelu", u1, w["ln2w"], w["ln2b"], B * L * 4, u1n)
        u2 = ops.gemm_tma(u1n.view(B * L * 4, 64), w["ct2"].bf16, w["ct2b"], act=2, out_dtype=bf)          # (B*L*4, 4*32), GELU'd
        hyper = torch.stack([self._mlp(self.output_hypernetworks_mlps[i], hs[:, 1 + i, :]) for i in range(self.num_mask_tokens)], dim=1).contiguous()
        m0, nm = (1, 3) if multimask_output else (0, 1)                                    # MaskDecoder.forward's mask_slice
        masks = torch.empty(B, nm, 4 * G, 4 * G, dtype=torch.float32, device=dev)
        _lib.call("sam6d_sam_mask_dot_range", u2, hyper, B, G, m0, nm, masks)
        iou = self._mlp(self.iou_prediction_head, hs[:, 0, :])
        return masks, iou[:, m0:m0 + nm].contiguous()

    @staticmethod
    def _mlp(mlp: _MLP, x):
        for i, layer in enumerate(mlp.layers):
            x = _lin(x, layer, relu=i < mlp.num_layers - 1)
        return x

    @torch.no_grad()
    def forward(self, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings, multimask_output=True):
        """-> (low-res logits (B,3,256,256), IoU (B,3)) of mask tokens 1..3, or (B,1,...), (B,1) of token 0 when not multimask_output"""
        return self.predict_masks(image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings, multimask_output)


# =====================================================================================================================
class Sam(nn.Module):
    mask_threshold: float = 0.0
    image_format: str = "RGB"

    def __init__(self, image_encoder, prompt_encoder, mask_decoder, pixel_mean=(123.675, 116.28, 103.53), pixel_std=(58.395, 57.12, 57.375)):
        super().__init__()
        self.image_encoder, self.prompt_encoder, self.mask_decoder = image_encoder, prompt_encoder, mask_decoder
        self.register_buffer("pixel_mean", torch.Tensor(pixel_mean).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.Tensor(pixel_std).view(-1, 1, 1), False)

    @property
    def device(self):
        return self.pixel_mean.device

    def preprocess(self, x):
        """sam.py:164-174: normalise, pad to 1024 x 1024 (elementwise plumbing on one frame)"""
        x = (x - self.pixel_mean) / self.pixel_std
        h, w = x.shape[-2:]
        s = self.image_encoder.img_size
        return torch.nn.functional.pad(x, (0, s - w, 0, s - h))

    @torch.no_grad()
    def postprocess_masks(self, masks: torch.Tensor, input_size: Tuple[int, ...], original_size: Tuple[int, ...]) -> torch.Tensor:
        """sam.py:133-162 (bilinear to img_size x img_size, crop to input_size, bilinear to original_size) as one kernel,
        `sam6d_sam_mask_upscale`: (B,C,S,S) low-res logits -> (B,C,H,W) f32 logits"""
        B, C, S = masks.shape[0], masks.shape[1], masks.shape[-1]
        H, W = int(original_size[0]), int(original_size[1])
        low = masks.float().contiguous()
        out = torch.empty(B, C, H, W, dtype=torch.float32, device=low.device)
        _lib.call("sam6d_sam_mask_upscale", low, B * C, S, self.image_encoder.img_size, int(input_size[0]), int(input_size[1]), H, W, out)
        return out

    def binarize_masks(self, masks: torch.Tensor, input_size: Tuple[int, ...], original_size: Tuple[int, ...]) -> torch.Tensor:
        """postprocess_masks(masks, ...) > mask_threshold without the logits: (B,C,S,S) -> (B,C,H,W) bool (`sam6d_sam_mask_binarize`)"""
        B, C, S = masks.shape[0], masks.shape[1], masks.shape[-1]
        H, W = int(original_size[0]), int(original_size[1])
        low = masks.float().contiguous()
        sel = torch.arange(B * C, dtype=torch.int32, device=low.device)
        out = torch.empty(B, C, H, W, dtype=torch.uint8, device=low.device)
        _lib.call("sam6d_sam_mask_binarize", low, sel, B * C, S, self.image_encoder.img_size, int(input_size[0]), int(input_size[1]), H, W,
                  self.mask_threshold, out)
        return out.view(torch.bool)


def build_sam_vit_h(precision="bf16") -> Sam:
    """build_sam.py:14-21,55-106 with this package's modules"""
    from .sam import build_image_encoder
    return Sam(build_image_encoder("vit_h", precision=precision), PromptEncoder(), MaskDecoder())


def build_sam_vit_l(precision="bf16") -> Sam:
    """build_sam.py:27-34,55-106 with this package's modules"""
    from .sam import build_image_encoder
    return Sam(build_image_encoder("vit_l", precision=precision), PromptEncoder(), MaskDecoder())


def build_sam_vit_b(precision="bf16") -> Sam:
    """build_sam.py:37-44,55-106 with this package's modules"""
    from .sam import build_image_encoder
    return Sam(build_image_encoder("vit_b", precision=precision), PromptEncoder(), MaskDecoder())


# build_sam.py:47-52
sam_model_registry = {
    "default": build_sam_vit_h,
    "vit_h": build_sam_vit_h,
    "vit_l": build_sam_vit_l,
    "vit_b": build_sam_vit_b,
}

# ISM/model/sam.py:17-21: the checkpoint file of each model type inside checkpoint_dir
pretrained_weight_dict = {
    "vit_l": "sam_vit_l_0b3195.pth",
    "vit_b": "sam_vit_b_01ec64.pth",
    "vit_h": "sam_vit_h_4b8939.pth",
}


def load_sam(model_type: str, checkpoint_dir: str, precision: str = "bf16") -> Sam:
    """drop-in for ISM/model/sam.py: load_sam (the hydra `model.segmentor_model.sam` target): builds `model_type` and loads
    `checkpoint_dir/pretrained_weight_dict[model_type]` strictly.  Returns the model on the CPU, like the reference."""
    if model_type not in pretrained_weight_dict:
        raise ValueError(f"unknown SAM model_type {model_type!r}: expected one of {sorted(pretrained_weight_dict)}")
    path = os.path.join(checkpoint_dir, pretrained_weight_dict[model_type])
    if not os.path.isfile(path):
        raise FileNotFoundError(f"SAM {model_type} checkpoint not found: {path} (expected {pretrained_weight_dict[model_type]} in {checkpoint_dir})")
    sam = sam_model_registry[model_type](precision)
    sam.load_state_dict(torch.load(path, map_location="cpu"), strict=True)
    return sam


def load_sam_predictor(model_type: str, checkpoint_dir: str, device, precision: str = "bf16") -> "SamPredictor":
    """drop-in for ISM/model/sam.py: load_sam_predictor: load_sam, move the model to `device`, wrap it in a SamPredictor"""
    sam = load_sam(model_type, checkpoint_dir, precision)
    sam.to(device=device)
    return SamPredictor(sam)


def preprocess_shape(oldh, oldw, long_side=1024) -> Tuple[int, int]:
    scale = long_side * 1.0 / max(oldh, oldw)
    return int(oldh * scale + 0.5), int(oldw * scale + 0.5)


class ResizeLongestSide:
    """utils/transforms.py: resize so the longest side is target_length, and the matching coordinate / box transforms"""

    def __init__(self, target_length: int) -> None:
        self.target_length = target_length

    def apply_image(self, image: np.ndarray) -> np.ndarray:
        """HxWxC uint8 -> resized, PIL bilinear (what torchvision's resize does on a PIL image)"""
        from PIL import Image
        nh, nw = self.get_preprocess_shape(image.shape[0], image.shape[1], self.target_length)
        return np.array(Image.fromarray(image).resize((nw, nh), Image.BILINEAR))

    def apply_coords(self, coords: np.ndarray, original_size: Tuple[int, ...]) -> np.ndarray:
        old_h, old_w = original_size
        new_h, new_w = self.get_preprocess_shape(original_size[0], original_size[1], self.target_length)
        coords = np.array(coords).astype(float)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes(self, boxes: np.ndarray, original_size: Tuple[int, ...]) -> np.ndarray:
        return self.apply_coords(np.asarray(boxes).reshape(-1, 2, 2), original_size).reshape(-1, 4)

    def apply_image_torch(self, image: torch.Tensor) -> torch.Tensor:
        """BxCxHxW float, antialiased bilinear (the reference notes this may differ from apply_image, which the model expects)"""
        target_size = self.get_preprocess_shape(image.shape[2], image.shape[3], self.target_length)
        return torch.nn.functional.interpolate(image, target_size, mode="bilinear", align_corners=False, antialias=True)

    def apply_coords_torch(self, coords: torch.Tensor, original_size: Tuple[int, ...]) -> torch.Tensor:
        old_h, old_w = original_size
        new_h, new_w = self.get_preprocess_shape(original_size[0], original_size[1], self.target_length)
        coords = coords.clone().to(torch.float)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes_torch(self, boxes: torch.Tensor, original_size: Tuple[int, ...]) -> torch.Tensor:
        return self.apply_coords_torch(boxes.reshape(-1, 2, 2), original_size).reshape(-1, 4)

    @staticmethod
    def get_preprocess_shape(oldh: int, oldw: int, long_side_length: int) -> Tuple[int, int]:
        return preprocess_shape(oldh, oldw, long_side_length)


@torch.no_grad()
def _encode_image(sam: Sam, transformed: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """the one image path of SamPredictor and CustomSamAutomaticMaskGenerator: (1,3,h,w) resized pixels on the device -> (features
    (1,256,64,64) f32, dense positional encoding as token rows (4096,256))"""
    features = sam.image_encoder(sam.preprocess(transformed.float())).float()
    return features, sam.prompt_encoder.dense_pe_rows()


def _resized_tensor(sam: Sam, transform: ResizeLongestSide, image: np.ndarray) -> torch.Tensor:
    """HxWx3 uint8 -> ResizeLongestSide.apply_image -> (1,3,h,w) uint8 on the model's device"""
    return torch.as_tensor(transform.apply_image(image), device=sam.device).permute(2, 0, 1).contiguous()[None]


class SamPredictor:
    """drop-in for segment_anything/predictor.py: one image embedding, then repeated prompt -> mask calls on it.  Prompts of one
    predict_torch call share the embedding and run as one batched decoder call."""

    def __init__(self, sam_model: Sam) -> None:
        self.model = sam_model
        self.transform = ResizeLongestSide(sam_model.image_encoder.img_size)
        self.reset_image()

    def set_image(self, image: np.ndarray, image_format: str = "RGB") -> None:
        assert image_format in ["RGB", "BGR"], f"image_format must be in ['RGB', 'BGR'], is {image_format}."
        if image_format != self.model.image_format:
            image = np.ascontiguousarray(image[..., ::-1])
        self.set_torch_image(_resized_tensor(self.model, self.transform, image), image.shape[:2])

    @torch.no_grad()
    def set_torch_image(self, transformed_image: torch.Tensor, original_image_size: Tuple[int, ...]) -> None:
        assert (len(transformed_image.shape) == 4 and transformed_image.shape[1] == 3
                and max(*transformed_image.shape[2:]) == self.model.image_encoder.img_size), \
            f"set_torch_image input must be BCHW with long side {self.model.image_encoder.img_size}."
        self.reset_image()
        self.original_size = tuple(original_image_size)
        self.input_size = tuple(transformed_image.shape[-2:])
        self.features, self.image_pe_rows = _encode_image(self.model, transformed_image)
        self.is_image_set = True

    def predict(self, point_coords: Optional[np.ndarray] = None, point_labels: Optional[np.ndarray] = None, box: Optional[np.ndarray] = None,
                mask_input: Optional[np.ndarray] = None, multimask_output: bool = True, return_logits: bool = False):
        """prompts in original-image pixels (numpy) -> (masks (C,H,W), iou (C), low-res logits (C,256,256)) as numpy"""
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        coords_torch, labels_torch, box_torch, mask_input_torch = None, None, None, None
        if point_coords is not None:
            assert point_labels is not None, "point_labels must be supplied if point_coords is supplied."
            point_coords = self.transform.apply_coords(point_coords, self.original_size)
            coords_torch = torch.as_tensor(point_coords, dtype=torch.float, device=self.device)[None, :, :]
            labels_torch = torch.as_tensor(point_labels, dtype=torch.int, device=self.device)[None, :]
        if box is not None:
            box = self.transform.apply_boxes(box, self.original_size)
            box_torch = torch.as_tensor(box, dtype=torch.float, device=self.device)[None, :]
        if mask_input is not None:
            mask_input_torch = torch.as_tensor(mask_input, dtype=torch.float, device=self.device)[None, :, :, :]
        masks, iou, low = self.predict_torch(coords_torch, labels_torch, box_torch, mask_input_torch, multimask_output, return_logits=return_logits)
        return masks[0].cpu().numpy(), iou[0].cpu().numpy(), low[0].cpu().numpy()

    @torch.no_grad()
    def predict_torch(self, point_coords: Optional[torch.Tensor], point_labels: Optional[torch.Tensor], boxes: Optional[torch.Tensor] = None,
                      mask_input: Optional[torch.Tensor] = None, multimask_output: bool = True, return_logits: bool = False):
        """prompts already in the resized frame (apply_coords_torch / apply_boxes_torch), batched over B ->
        (masks (B,C,H,W) bool, or f32 logits with return_logits; iou (B,C); low-res logits (B,C,256,256))"""
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        points = (point_coords, point_labels) if point_coords is not None else None
        sparse, dense = self.model.prompt_encoder(points=points, boxes=boxes, masks=mask_input)
        low, iou = self.model.mask_decoder(self.features, self.image_pe_rows, sparse, dense, multimask_output)
        if return_logits:
            masks = self.model.postprocess_masks(low, self.input_size, self.original_size)
        else:
            masks = self.model.binarize_masks(low, self.input_size, self.original_size)
        return masks, iou, low

    def get_image_embedding(self) -> torch.Tensor:
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) to generate an embedding.")
        assert self.features is not None, "Features must exist if an image has been set."
        return self.features

    @property
    def device(self) -> torch.device:
        return self.model.device

    def reset_image(self) -> None:
        self.is_image_set = False
        self.features = None
        self.image_pe_rows = None
        self.original_size = None
        self.input_size = None
        self.orig_h = self.orig_w = self.input_h = self.input_w = None


def build_point_grid(n_per_side: int) -> np.ndarray:
    offset = 1 / (2 * n_per_side)
    pts = np.linspace(offset, 1 - offset, n_per_side)
    return np.stack([np.tile(pts[None, :], (n_per_side, 1)), np.tile(pts[:, None], (1, n_per_side))], axis=-1).reshape(-1, 2)


class CustomSamAutomaticMaskGenerator:
    """generate_masks(image (H,W,3) uint8) -> {"masks": (N,H,W) float 0/1, "boxes": (N,4) float xyxy} like ISM/model/sam.py:103-155
    (single crop: crop_n_layers = 0, the SAM-6D configuration)."""

    def __init__(self, sam: Sam, min_mask_region_area=0, points_per_batch=64, stability_score_thresh=0.85, box_nms_thresh=0.7,
                 crop_overlap_ratio=512 / 1500, segmentor_width_size=None, pred_iou_thresh=0.88, points_per_side=32,
                 stability_score_offset=1.0):
        if min_mask_region_area:
            raise NotImplementedError("min_mask_region_area > 0 (cv2 connected components) is not used by SAM-6D")
        self.sam, self.points_per_batch, self.points_per_side = sam, points_per_batch, points_per_side
        self.stability_score_thresh, self.box_nms_thresh, self.pred_iou_thresh = stability_score_thresh, box_nms_thresh, pred_iou_thresh
        self.stability_score_offset, self.segmentor_width_size = stability_score_offset, segmentor_width_size
        self.features = None

    # ---- SamPredictor.set_image ----------------------------------------------------------------------------------------------
    @torch.no_grad()
    def set_image(self, image: np.ndarray):
        """ResizeLongestSide.apply_image (PIL bilinear, host: the reference does the same) -> normalise, pad, image encoder; the
        same helpers as SamPredictor.set_image"""
        x = _resized_tensor(self.sam, ResizeLongestSide(self.sam.image_encoder.img_size), image)
        self.original_size, self.input_size = tuple(image.shape[:2]), tuple(x.shape[-2:])
        self.features, self.image_pe_rows = _encode_image(self.sam, x)
        return self.features

    # ---- one batch of point prompts ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def process_batch(self, points: np.ndarray):
        """_process_batch (automatic_mask_generator.py:265-321) -> (kept masks (k,H,W) u8, boxes (k,4) i64, iou (k) f32, low-res
        logits (n*3,256,256), iou of all n*3, stats (n*3,8))"""
        H, W = self.original_size
        nh, nw = self.input_size
        dev = self.sam.device
        c = points.astype(float).copy()
        c[..., 0] *= nw / W
        c[..., 1] *= nh / H
        pts = torch.as_tensor(c, device=dev)[:, None, :]
        labels = torch.ones(pts.shape[0], 1, dtype=torch.int, device=dev)
        sparse, dense = self.sam.prompt_encoder(points=(pts, labels))
        low, iou = self.sam.mask_decoder(self.features, self.image_pe_rows, sparse, dense, True)
        n = low.shape[0] * 3
        low = low.view(n, low.shape[-2], low.shape[-1])
        stats = torch.empty(n, 8, dtype=torch.int32, device=dev)
        _lib.call("sam6d_sam_mask_stats", low, n, low.shape[-1], self.sam.image_encoder.img_size, nh, nw, H, W, self.sam.mask_threshold,
                  self.stability_score_offset, stats)
        iou_f = iou.reshape(-1)
        st = stats.cpu()
        iou_h = iou_f.cpu()
        stab = st[:, 0].float() / st[:, 1].float()                                   # intersections / unions (amg.py:156-176)
        keep = (iou_h > self.pred_iou_thresh) & (stab >= self.stability_score_thresh)
        sel = torch.nonzero(keep).flatten()
        boxes = st[sel][:, 2:6].long()
        empty = (boxes[:, 2] < boxes[:, 0]) | (boxes[:, 3] < boxes[:, 1])
        boxes[empty] = 0
        masks = torch.empty(len(sel), H, W, dtype=torch.uint8, device=dev)
        if len(sel):
            sel_d = sel.to(device=dev, dtype=torch.int32)
            _lib.call("sam6d_sam_mask_binarize", low, sel_d, len(sel), low.shape[-1], self.sam.image_encoder.img_size, nh, nw, H, W,
                      self.sam.mask_threshold, masks)
        return masks, boxes.to(dev), iou_f[sel.to(dev)], low, iou_f, stats

    @staticmethod
    def nms(boxes: torch.Tensor, scores: torch.Tensor, thr: float) -> torch.Tensor:
        """torchvision.ops.batched_nms with one category: kept indices by decreasing score"""
        if boxes.shape[0] == 0:
            return torch.zeros(0, dtype=torch.long, device=boxes.device)
        order = torch.argsort(scores, descending=True, stable=True)
        b = boxes[order].float().contiguous()
        keep = torch.empty(b.shape[0], dtype=torch.uint8, device=b.device)
        _lib.call("sam6d_sam_nms", b, None, b.shape[0], thr, keep)
        return order[keep.bool()]

    @torch.no_grad()
    def _generate_masks(self, image: np.ndarray) -> Dict[str, Any]:
        H, W = image.shape[:2]
        self.set_image(image)
        pts = build_point_grid(self.points_per_side) * np.array([W, H])[None, :]
        ms, bs, ss = [], [], []
        for i in range(0, len(pts), self.points_per_batch):
            m, b, s = self.process_batch(pts[i:i + self.points_per_batch])[:3]
            ms.append(m); bs.append(b); ss.append(s)
        masks, boxes, iou = torch.cat(ms), torch.cat(bs), torch.cat(ss)
        keep = self.nms(boxes, iou, self.box_nms_thresh)
        return {"masks": masks[keep].bool(), "boxes": boxes[keep], "iou_preds": iou[keep]}

    @torch.no_grad()
    def generate_masks(self, image: np.ndarray) -> Dict[str, Any]:
        orig = image.shape[:2]
        if self.segmentor_width_size is not None and self.segmentor_width_size != image.shape[1]:
            import cv2
            image = cv2.resize(image.copy(), (self.segmentor_width_size, int(self.segmentor_width_size * orig[0] / orig[1])))
        d = self._generate_masks(image)
        masks, boxes = d["masks"].float(), d["boxes"].float()
        if self.segmentor_width_size is not None:                                   # postprocess_resize (ISM/model/sam.py:83-100)
            if masks.shape[-2:] != orig and masks.shape[0]:
                masks = torch.nn.functional.interpolate(masks.unsqueeze(1), size=orig, mode="bilinear", align_corners=False)[:, 0]
            boxes = boxes * (orig[1] / self.segmentor_width_size)
            boxes[:, [0, 2]] = torch.clamp(boxes[:, [0, 2]], 0, orig[1] - 1)
            boxes[:, [1, 3]] = torch.clamp(boxes[:, [1, 3]], 0, orig[0] - 1)
        return {"masks": masks, "boxes": boxes}
