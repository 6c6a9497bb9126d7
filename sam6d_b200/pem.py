"""Pose Estimation Model matching path on H100 kernels -- drop-in for the reference's model classes.

Class names, constructor arguments, sub-module / parameter names (hence `state_dict` keys) and the `forward` contracts
mirror the reference:
    Net                         PEM/model/pose_estimation_model.py:11-53
    GeometricStructureEmbedding PEM/model/transformer.py:286-349
    GeometricTransformer        PEM/model/transformer.py:469-513
    SparseToDenseTransformer    PEM/model/transformer.py:613-673
    CoarsePointMatching         PEM/model/coarse_point_matching.py:14-81
    FinePointMatching           PEM/model/fine_point_matching.py:12-126
so `sam-6d-pem-base.pth` loads unchanged.  The torch modules here are parameter containers only: every forward runs
hand-written sm_90a kernels through the C ABI (sam6d_b200/ops.py); inference only (the reference's training branches --
losses, pose-noise augmentation -- are out of scope), and there is no CPU path.
"""
import math
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn as nn

from . import ops
from .layers import _W, _f32, _gemm, _Packed, _param_key, PRECISIONS

NUM_HEADS = 4  # hard-coded in the reference (coarse_point_matching.py:31, fine_point_matching.py:29)

# PRECISIONS (layers.py): in "bf16" the geometric embedding is stored in bf16 as well.  Index-valued results (FPS, ball
# query, labels) and the pose solvers are identical in both modes.
# bf16 self-attention: TMA + wgmma score stream into padded planes (csrc/rpe_tc.cu); bench.py reads these to name the kernels it times
RPE_TC = True
PADDED_BIAS = True
# bf16 path: the geometric embedding by table interpolation (csrc/geo_lut.cu)
GEO_LUT_INV_H = 8.0            # table step 1/8 index unit
GEO_LUT_D_MAX = 32.0           # distance indices below this come from the table: 6.4 object radii (the reference's input builder
                               # keeps scene points within 1.2 radii of the mask centroid: indices <= 12)


def _cfg(cfg, **defaults):
    """accept gorilla Config / dict / namespace like the reference's cfg objects"""
    if isinstance(cfg, dict):
        cfg = SimpleNamespace(**cfg)
    for k, v in defaults.items():
        if not hasattr(cfg, k):
            setattr(cfg, k, v)
    return cfg


# =====================================================================================================================
# parameter containers with the reference's names
# =====================================================================================================================
class _MHAParams(nn.Module):
    def __init__(self, d_model, rpe: bool):
        super().__init__()
        self.proj_q = nn.Linear(d_model, d_model)
        self.proj_k = nn.Linear(d_model, d_model)
        self.proj_v = nn.Linear(d_model, d_model)
        if rpe:
            self.proj_p = nn.Linear(d_model, d_model)


class _AttentionLayerParams(nn.Module):
    def __init__(self, d_model, rpe: bool):
        super().__init__()
        self.attention = _MHAParams(d_model, rpe)
        self.linear = nn.Linear(d_model, d_model)
        self.norm = nn.LayerNorm(d_model)


class _AttentionOutputParams(nn.Module):
    def __init__(self, d_model):
        super().__init__()
        self.expand = nn.Linear(d_model, d_model * 2)
        self.squeeze = nn.Linear(d_model * 2, d_model)
        self.norm = nn.LayerNorm(d_model)


class _TransformerLayerParams(nn.Module):
    def __init__(self, d_model, rpe: bool):
        super().__init__()
        self.attention = _AttentionLayerParams(d_model, rpe)
        self.output = _AttentionOutputParams(d_model)


def _pair(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The scene cloud and the template cloud go through the same weights in most layers, so the modules run them as one
    (2B, ...) batch [a ; b].  That is a view when a and b are the two halves of one allocation (Net.forward builds them that
    way) and a concatenated copy otherwise (the reference API passes them as separate arguments): the kernels see the same
    batch either way, so results do not depend on how the caller allocated the clouds."""
    if a.shape != b.shape or a.dtype != b.dtype:
        raise ValueError(f"the two clouds must have equal shapes and dtypes: {tuple(a.shape)} {a.dtype}, {tuple(b.shape)} {b.dtype}")
    if (a.is_contiguous() and b.is_contiguous() and a.device == b.device
            and a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()
            and b.storage_offset() == a.storage_offset() + a.numel()):
        return torch.as_strided(a, (2 * a.numel(),), (1,), a.storage_offset()).view(2 * a.shape[0], *a.shape[1:])
    return torch.cat([a, b])


# ---------------------------------------------------------------------------------------------------------------------
# shared token-layer math
# ---------------------------------------------------------------------------------------------------------------------
def _attn_tail(x2d: torch.Tensor, hid: torch.Tensor, lw) -> torch.Tensor:
    """AttentionLayer / RPEAttentionLayer tail + AttentionOutput (transformer.py:176-197, 435-438), fp32:
       y = LN(linear(hid) + x);  out = LN(y + squeeze(relu(expand(y))))"""
    y = ops.gemm(hid, lw["wo"].f32, lw["bo"], residual=x2d)
    y = ops.layernorm(y, lw["g1"], lw["b1"])
    h = ops.gemm(y, lw["we"].f32, lw["be"], relu=True)
    z = ops.gemm(h, lw["ws"].f32, lw["bs"], residual=y)
    return ops.layernorm(z, lw["g2"], lw["b2"])


def _pack_tail(layer: nn.Module) -> Dict[str, torch.Tensor]:
    """the tail weights of a _TransformerLayerParams or _LinearTransformerLayerParams (same attention.linear/norm, output.*)"""
    a, o = layer.attention, layer.output
    return dict(wo=_W(a.linear.weight), bo=_f32(a.linear.bias), g1=_f32(a.norm.weight), b1=_f32(a.norm.bias),
                we=_W(o.expand.weight), be=_f32(o.expand.bias), ws=_W(o.squeeze.weight), bs=_f32(o.squeeze.bias),
                g2=_f32(o.norm.weight), b2=_f32(o.norm.bias))


def _tail_bf16(x2d: torch.Tensor, hid: torch.Tensor, lw, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """_attn_tail for the bf16 token stream as one kernel (csrc/tail_tc.cu): x2d, hid, out (M,256) bf16"""
    return ops.transformer_tail_bf16(hid, x2d, lw["wo"].bf16, lw["bo"], lw["g1"], lw["b1"], lw["we"].bf16, lw["be"],
                                     lw["ws"].bf16, lw["bs"], lw["g2"], lw["b2"], out=out)


class GeometricTransformer(nn.Module):
    """blocks = ['self', 'cross'] with parallel=False, as instantiated by the reference (coarse_point_matching.py:28-35,
    transformer.py:633-641).  forward(feats0, embeddings0, feats1, embeddings1) -> (feats0, feats1)."""

    def __init__(self, blocks, d_model, num_heads, dropout=None, activation_fn='ReLU', return_attention_scores=False,
                 parallel=False):
        super().__init__()
        if list(blocks) != ['self', 'cross'] or parallel or return_attention_scores or dropout:
            raise ValueError("sam6d_b200.GeometricTransformer supports the configuration SAM-6D uses: "
                             "blocks=['self','cross'], parallel=False, dropout=None, no attention-score output")
        if activation_fn != 'ReLU' or num_heads != NUM_HEADS or d_model != 256:
            raise ValueError("sam6d_b200 kernels are built for d_model=256, num_heads=4, ReLU")
        self.blocks = list(blocks)
        self.d_model, self.num_heads = d_model, num_heads
        self.layers = nn.ModuleList([_TransformerLayerParams(d_model, rpe=True), _TransformerLayerParams(d_model, rpe=False)])
        self._packed = _Packed()
        self.precision = "fp32"

    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        C, H = self.d_model, self.num_heads
        d = C // H
        sa = self.layers[0].attention.attention
        wq, bq = _f32(sa.proj_q.weight), _f32(sa.proj_q.bias)
        wp = _f32(sa.proj_p.weight)
        # u_h = W_p,h^T (W_q,h x + b_q,h): fold proj_p into the query side (one (C x C) matrix per head)
        mu = [wp[h * d:(h + 1) * d, :].t().double() @ wq[h * d:(h + 1) * d, :].double() for h in range(H)]
        cu = [wp[h * d:(h + 1) * d, :].t().double() @ bq[h * d:(h + 1) * d].double() for h in range(H)]
        w_self = torch.cat([wq, _f32(sa.proj_k.weight), _f32(sa.proj_v.weight)] + [m.float() for m in mu], dim=0)
        b_self = torch.cat([bq, _f32(sa.proj_k.bias), _f32(sa.proj_v.bias)] + [c.float() for c in cu], dim=0)
        ca = self.layers[1].attention.attention
        return dict(
            w_self=_W(w_self), b_self=b_self.contiguous(), tail_self=_pack_tail(self.layers[0]),
            # bf16 self-attention outside rpe_tc's reach (_self_bf16): q|k|v as one bf16 GEMM, the folded rel-pos queries u
            # as a second (fp32) one
            w_qkv=_W(w_self[:3 * C]), b_qkv=b_self[:3 * C].contiguous(), w_u=_W(w_self[3 * C:]), b_u=b_self[3 * C:].contiguous(),
            wq_c=_W(ca.proj_q.weight), bq_c=_f32(ca.proj_q.bias),
            wkv_c=_W(torch.cat([_f32(ca.proj_k.weight), _f32(ca.proj_v.weight)], dim=0)),
            bkv_c=torch.cat([_f32(ca.proj_k.bias), _f32(ca.proj_v.bias)], dim=0).contiguous(),
            # cloud 1 is the memory of the first cross layer and the query of the second: one projection [k | q | v]
            wkqv_c=_W(torch.cat([_f32(ca.proj_k.weight), _f32(ca.proj_q.weight), _f32(ca.proj_v.weight)], dim=0)),
            bkqv_c=torch.cat([_f32(ca.proj_k.bias), _f32(ca.proj_q.bias), _f32(ca.proj_v.bias)], dim=0).contiguous(),
            tail_cross=_pack_tail(self.layers[1]))

    # ---- fp32 (precision="fp32"): CUDA-core kernels, fp32 storage
    def _self_layer(self, x: torch.Tensor, emb: torch.Tensor, w) -> torch.Tensor:
        B, S, C = x.shape
        x2d = x.reshape(B * S, C)
        qkvu = ops.gemm(x2d, w["w_self"].f32, w["b_self"])                       # (B*S, q|k|v|u0..u3)
        sp = ops.rpe_scores(emb, qkvu[:, 3 * C:])                                  # (B,H,S,S)
        hid = torch.empty(B * S, C, dtype=torch.float32, device=x.device)
        qkv = qkvu.view(B, S, -1)
        ops.mha(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:3 * C], sp, 1.0 / math.sqrt(C // NUM_HEADS), hid.view(B, S, C))
        return _attn_tail(x2d, hid, w["tail_self"]).view(B, S, C)

    def _cross_layer(self, x: torch.Tensor, mem: torch.Tensor, w) -> torch.Tensor:
        B, S, C = x.shape
        Sm = mem.shape[1]
        x2d = x.reshape(B * S, C)
        q = ops.gemm(x2d, w["wq_c"].f32, w["bq_c"])
        kv = ops.gemm(mem.reshape(B * Sm, C), w["wkv_c"].f32, w["bkv_c"]).view(B, Sm, 2 * C)
        hid = torch.empty(B * S, C, dtype=torch.float32, device=x.device)
        ops.mha(q.view(B, S, C), kv[..., :C], kv[..., C:], None, 1.0 / math.sqrt(C // NUM_HEADS), hid.view(B, S, C))
        return _attn_tail(x2d, hid, w["tail_cross"]).view(B, S, C)

    # ---- bf16 token stream (precision="bf16"): every Linear is the persistent TMA GEMM, the residual stream, LayerNorm
    # inputs/outputs and the attention output are bf16, accumulation and statistics fp32.
    def _self_bf16(self, x, emb, w):
        B, S, C = x.shape
        d = C // NUM_HEADS
        x2d = x.view(B * S, C)
        if S <= 200 and emb.dtype == torch.bfloat16:
            # ONE projection launch: (q | k) rows, V^T, and the folded rel-pos queries u as bf16 rows = the B operand of the TMA /
            # wgmma stream over E (csrc/rpe_tc.cu)
            qk, vt, u = ops.gemm_tma_vt2(x2d, w["w_self"].bf16, w["b_self"], 2 * C, 3 * C, S)
            # score planes with 16-key padded rows: the attention kernel streams them with 16-byte cp.async copies
            sp = ops.rpe_scores_tc_padded(emb, u)
            hid = ops.attn_tc_padded_bias(qk, 0, qk, C, vt, B, NUM_HEADS, S, S, d, 1.0 / math.sqrt(d), sp)
            return _tail_bf16(x2d, hid, w["tail_self"]).view(B, S, C)
        qk, vt = ops.gemm_tma_vt(x2d, w["w_qkv"].bf16, w["b_qkv"], 2 * C, S)                        # (B*S, q|k) and V^T
        u = ops.gemm_tma(x2d, w["w_u"].bf16, w["b_u"])                                              # (B*S, 4*C) fp32
        sp = ops.rpe_scores(emb, u)
        hid = ops.attn_tc(qk, 0, qk, C, vt, B, NUM_HEADS, S, S, d, 1.0 / math.sqrt(d), bias=sp, out_dtype=torch.bfloat16)
        return _tail_bf16(x2d, hid, w["tail_self"]).view(B, S, C)

    def _forward_bf16(self, f, emb, w):
        """f (2B,S,C) bf16 = [cloud 0 ; cloud 1], emb (2B,S,S,256) -> same layout"""
        B, S, C = f.shape[0] // 2, f.shape[1], f.shape[2]
        d = C // NUM_HEADS
        scale = 1.0 / math.sqrt(d)
        f = self._self_bf16(f, emb, w)
        out = torch.empty_like(f)
        x0, x1 = f[:B].view(B * S, C), f[B:].view(B * S, C)
        # cross layer 0: cloud 0 attends to cloud 1.  ONE projection [k | q | v] over both clouds: cloud 0's queries, cloud 1's keys
        # / values, and cloud 1's queries for the second layer (cloud 0's keys / values of the old features are not used)
        kq, vt_all = ops.gemm_tma_vt(f.view(2 * B * S, C), w["wkqv_c"].bf16, w["bkqv_c"], 2 * C, S, slot=1)
        kq1, vt1 = kq[B * S:], vt_all[B * C:]
        hid = ops.attn_tc(kq, C, kq1, 0, vt1, B, NUM_HEADS, S, S, d, scale, out_dtype=torch.bfloat16)
        _tail_bf16(x0, hid, w["tail_cross"], out=out[:B].view(B * S, C))
        # cross layer 1: cloud 1 attends to the updated cloud 0 (sequential, transformer.py:505-507)
        k0, vt0 = ops.gemm_tma_vt(out[:B].view(B * S, C), w["wkv_c"].bf16, w["bkv_c"], C, S, slot=2)
        hid = ops.attn_tc(kq1, C, k0, 0, vt0, B, NUM_HEADS, S, S, d, scale, out_dtype=torch.bfloat16)
        _tail_bf16(x1, hid, w["tail_cross"], out=out[B:].view(B * S, C))
        return out

    @torch.no_grad()
    def forward(self, feats0, embeddings0, feats1, embeddings1, masks0=None, masks1=None):
        if masks0 is not None or masks1 is not None:
            raise NotImplementedError("key masks are never used on the SAM-6D inference path")
        w = self._weights()
        B = feats0.shape[0]
        # both clouds share the self-attention weights: one batch of 2B through every kernel of the layer
        f, emb = _pair(feats0, feats1), _pair(embeddings0, embeddings1)
        if self.precision == "bf16":
            f = self._forward_bf16(f.to(torch.bfloat16).contiguous(), emb, w)
            return f[:B], f[B:]
        f = self._self_layer(f, emb, w)
        feats0, feats1 = f[:B], f[B:]
        feats0 = self._cross_layer(feats0, feats1, w)
        feats1 = self._cross_layer(feats1, feats0, w)      # sequential: sees the updated feats0 (transformer.py:505-507)
        return feats0, feats1


# =====================================================================================================================
class _SinusoidalBuffer(nn.Module):
    def __init__(self, d_model):
        super().__init__()
        div_indices = torch.arange(0, d_model, 2).float()
        self.register_buffer('div_term', torch.exp(div_indices * (-math.log(10000.0) / d_model)))


class GeometricStructureEmbedding(nn.Module):
    """forward(points (B,S,3)) -> (B,S,S,hidden_dim) pair embedding; cfg: sigma_d, sigma_a, angle_k, reduction_a, hidden_dim."""

    def __init__(self, cfg):
        super().__init__()
        cfg = _cfg(cfg)
        self.sigma_d, self.sigma_a, self.angle_k = cfg.sigma_d, cfg.sigma_a, cfg.angle_k
        self.factor_a = 180.0 / (self.sigma_a * math.pi)
        if cfg.reduction_a != 'max' or cfg.angle_k != 3 or cfg.hidden_dim != 256:
            raise ValueError("sam6d_b200 kernels are built for reduction_a='max', angle_k=3, hidden_dim=256")
        self.embedding = _SinusoidalBuffer(cfg.hidden_dim)
        self.proj_d = nn.Linear(cfg.hidden_dim, cfg.hidden_dim)
        self.proj_a = nn.Linear(cfg.hidden_dim, cfg.hidden_dim)
        self._packed = _Packed()
        self.precision = "fp32"

    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        w = dict(div=_f32(self.embedding.div_term), waT=_f32(self.proj_a.weight).t().contiguous(),
                 wdT=_f32(self.proj_d.weight).t().contiguous(), wd_bf=_f32(self.proj_d.weight).to(torch.bfloat16).contiguous(),
                 bias=(_f32(self.proj_a.bias) + _f32(self.proj_d.bias)).contiguous())
        w.update(self._tables(w))
        return w

    def _tables(self, w):
        """g_a(x) = W_a emb(x) on [0, 180 / sigma_a] and g_d(x) = W_d emb(x) + (b_a + b_d) on [0, GEO_LUT_D_MAX], step
        1 / GEO_LUT_INV_H, evaluated in float64 from the fp32 weights and stored in bf16 (csrc/geo_lut.cu interpolates them)"""
        div = w["div"].double()

        def table(weight, x_max, bias=None):
            n = int(math.ceil(x_max * GEO_LUT_INV_H)) + 1
            om = (torch.arange(n, dtype=torch.float64, device=div.device) / GEO_LUT_INV_H)[:, None] * div[None, :]
            emb = torch.stack([torch.sin(om), torch.cos(om)], dim=2).reshape(n, -1)      # interleaved (sin, cos) per frequency
            g = emb @ weight.detach().double().t()
            if bias is not None:
                g = g + bias.double()
            return g.to(torch.float32).to(torch.bfloat16).contiguous()

        return dict(tab_a=table(self.proj_a.weight, 180.0 / self.sigma_a), tab_d=table(self.proj_d.weight, GEO_LUT_D_MAX, w["bias"]),
                    wdT_bf=_f32(self.proj_d.weight).t().contiguous().to(torch.bfloat16).contiguous())

    @torch.no_grad()
    def get_embedding_indices(self, points):
        T = ops.geo_indices(points.contiguous(), self.sigma_d, self.factor_a)
        return T[..., 3], T[..., :3]

    @torch.no_grad()
    def forward(self, points):
        w = self._weights()
        T = ops.geo_indices(points.contiguous(), self.sigma_d, self.factor_a)
        if self.precision == "bf16":
            # distances of row 0 / column 0 (the background point of SAM-6D: far outside the table) go through the exact
            # tensor-core projection: 2 S values per cloud
            far = ops.geo_embed_dist_tc(torch.stack([T[:, 0, :, :], T[:, :, 0, :]], dim=1).contiguous(), w["div"], w["wd_bf"], w["bias"])
            return ops.geo_embed_lut(T, w["tab_a"], GEO_LUT_INV_H, w["tab_d"], GEO_LUT_INV_H, far, w["div"], w["wdT_bf"], w["bias"])
        return ops.geo_embed_f32(T, w["div"], w["waT"], w["wdT"], w["bias"])


# =====================================================================================================================
# pose solvers (PEM/utils/model_utils.py)
# =====================================================================================================================
def sample_pts_feats(pts, feats, npoint=2048, return_index=False):
    """model_utils.py:53-66 (FPS + two gathers, channel-last)."""
    idx = ops.furthest_point_sampling(pts.contiguous(), npoint)
    p = ops.gather_rows(pts.contiguous(), idx)
    # a bf16 feature matrix (Net.forward's stacked bf16 copy) comes back as fp32 rows -- exact, and what the coarse in_proj reads
    f = ops.gather_rows_bf16_f32(feats.contiguous(), idx) if feats.dtype == torch.bfloat16 else ops.gather_rows(feats.contiguous(), idx)
    return (p, f, idx) if return_index else (p, f)


def compute_feature_similarity(feat1, feat2, type='cosine', temp=1.0, normalize_feat=True, precision="fp32"):
    """model_utils.py:114-136 -> (B,N,M) = normalize(f1) normalize(f2)^T / temp."""
    if type != 'cosine':
        raise NotImplementedError("SAM-6D uses sim_type='cosine'")
    B, N, C = feat1.shape
    M = feat2.shape[1]
    ld = (M + 3) // 4 * 4                      # rows padded to 16 bytes so the epilogue can use full-line vector stores
    store = torch.empty(B, N, ld, dtype=torch.float32, device=feat1.device)
    if precision == "bf16":
        # normalised bf16 tokens -> persistent TMA GEMM over all proposals (tiles that run past a proposal's rows are masked)
        f1 = ops.l2norm_rows_bf16(feat1.contiguous()) if normalize_feat else feat1.contiguous().to(torch.bfloat16)
        f2 = ops.l2norm_rows_bf16(feat2.contiguous()) if normalize_feat else feat2.contiguous().to(torch.bfloat16)
        ops.gemm_tma_batched(f1, f2, store[:, :, :M], alpha=1.0 / temp)
    else:
        f1 = ops.l2norm_rows(feat1.contiguous()) if normalize_feat else feat1.contiguous()
        f2 = ops.l2norm_rows(feat2.contiguous()) if normalize_feat else feat2.contiguous()
        ops.gemm(f1, f2, out=store[:, :, :M], alpha=1.0 / temp)
    return store[:, :, :M]                     # (B,N,M) like the reference; dense rows, row stride ld


def compute_coarse_Rt(atten, pts1, pts2, model_pts=None, n_proposal1=6000, n_proposal2=300, rand=None, return_scores=False,
                      n_hypotheses=1, min_angle=30.0, min_dist=0.2, symmetries=None):
    """model_utils.py:187-246.  `rand` (B, 3*n_proposal1) overrides the torch.rand draw (used by the parity tests to feed the
    reference and this implementation the same uniforms); by default the call is the reference's own
    torch.rand(B, n_proposal1*3, device=device), so the Philox stream position matches.
    n_hypotheses = K > 1 (not in the reference) appends the K mutually distinct hypotheses of ops.coarse_pick_distinct (at least
    min_angle degrees or min_dist radius-normalised units apart) to the return values: R (B,K,3,3), t (B,K,3), score (B,K),
    valid (B,K) u8, count (B) i32, slot 0 being the returned R, t.  symmetries = (symR (S,3,3), symt (S,3) metres, sym_range (B,2)
    i32, radius (B)): with K > 1 two hypotheses are then distinct only when they are so from every symmetric copy of each other
    (ops.coarse_pick_distinct_sym)."""
    B = pts1.shape[0]
    if model_pts is None:
        model_pts = pts2
    W, w1 = ops.coarse_assign(atten.contiguous())   # (B,197,197): the copy out of the padded rows is 5 MB
    if rand is None:
        rand = torch.rand(B, n_proposal1 * 3, device=pts1.device)
    idx = ops.coarse_sample(W, rand.contiguous())
    Rt, resid = ops.coarse_hypotheses(idx, pts1.contiguous(), pts2.contiguous())
    top = ops.topk_smallest(resid, n_proposal2)
    R, t, scores = ops.coarse_select(Rt, top, pts1.contiguous(), w1, model_pts.contiguous())
    if n_hypotheses > 1 and symmetries is not None:
        hyp = ops.coarse_pick_distinct_sym(Rt, top, scores, n_hypotheses, min_angle, min_dist, *symmetries)
    else:
        hyp = ops.coarse_pick_distinct(Rt, top, scores, n_hypotheses, min_angle, min_dist) if n_hypotheses > 1 else ()
    if return_scores:
        return (R, t, scores) + hyp  # (B, n_proposal2) selection scores of the retained hypotheses
    return (R, t) + hyp


def compute_fine_Rt(atten, pts1, pts2, model_pts=None, dis_thres=0.15, temp=0.1, radius=None, check_bound=True):
    """model_utils.py:250-283.  Returns (R, t, pose_score); with `radius` also t * (radius + 1e-6).
    `atten` must be a cosine-similarity matrix divided by `temp` (|atten| <= 1/temp): the assignment kernels use the fixed
    soft-max shift 1/temp instead of a per-row / per-column maximum pass, which is exact for such scores and overflows for
    unbounded ones -- so out-of-range input raises instead of silently returning inf / NaN (`check_bound=False` skips that
    host read-back for callers whose scores are cosines by construction: FinePointMatching)."""
    if model_pts is None:
        model_pts = pts2
    bound = 1.0 / temp
    if check_bound and float(atten.abs().max()) > bound * (1.0 + 1e-3):
        raise ValueError(f"compute_fine_Rt: |atten| exceeds 1/temp = {bound:g}; the CUDA path handles cosine scores "
                         "(sim_type='cosine', normalize_feat=True) only")
    pts1, pts2 = pts1.contiguous(), pts2.contiguous()
    lab1, _, wts, pred = ops.fine_assign(atten, pts2, shift=1.0 / temp)
    R, t = ops.weighted_procrustes(pred, pts1, wts, 0.0, 1e-5)
    rad = radius if radius is not None else torch.ones(pts1.shape[0], device=pts1.device) - 1e-6
    score, t_scaled = ops.pose_score(pts1, lab1, R, t, model_pts.contiguous(), rad.contiguous(), dis_thres)
    return (R, t, score) if radius is None else (R, t, score, t_scaled)


# =====================================================================================================================
class CoarsePointMatching(nn.Module):
    """forward(p1, f1, geo1, p2, f2, geo2, radius, end_points) -> end_points with init_R, init_t."""

    def __init__(self, cfg, return_feat=False):
        super().__init__()
        self.cfg = _cfg(cfg)
        self.return_feat = return_feat
        self.nblock = self.cfg.nblock
        self.in_proj = nn.Linear(self.cfg.input_dim, self.cfg.hidden_dim)
        self.out_proj = nn.Linear(self.cfg.hidden_dim, self.cfg.out_dim)
        self.bg_token = nn.Parameter(torch.randn(1, 1, self.cfg.hidden_dim) * .02)
        self.transformers = nn.ModuleList([
            GeometricTransformer(blocks=['self', 'cross'], d_model=self.cfg.hidden_dim, num_heads=4, dropout=None,
                                 activation_fn='ReLU', return_attention_scores=False) for _ in range(self.nblock)])
        self._packed = _Packed()
        self.precision = "fp32"

    def _weights(self):
        return self._packed.get(lambda: dict(w_in=_W(self.in_proj.weight), b_in=_f32(self.in_proj.bias), w_out=_W(self.out_proj.weight),
                                             b_out=_f32(self.out_proj.bias)), self.in_proj, self.out_proj)

    def _embed(self, f):
        B, n, C = f.shape
        w = self._weights()
        H = self.cfg.hidden_dim
        if self.precision == "bf16":                          # the sparse token stream is bf16 in this mode
            out = torch.empty(B, n + 1, H, dtype=torch.bfloat16, device=f.device)
            out[:, 0, :] = self.bg_token.detach().reshape(1, -1).to(torch.bfloat16)
            ops.gemm_tc(f, w["w_in"].bf16, w["b_in"], out=out[:, 1:, :])
            return out
        out = torch.empty(B, n + 1, H, dtype=torch.float32, device=f.device)
        out[:, 0, :] = self.bg_token.detach().reshape(1, -1)
        _gemm(self.precision, f, w["w_in"], w["b_in"], out=out[:, 1:, :])
        return out

    @torch.no_grad()
    def forward(self, p1, f1, geo1, p2, f2, geo2, radius, end_points, rand=None, hypotheses=(1, 30.0, 0.2)):
        """hypotheses = (K, min_angle, min_dist): with K > 1 end_points also gets hyp_init_R (B,K,3,3), hyp_init_t (B,K,3) and
        hyp_valid (B,K) u8 of compute_coarse_Rt's distinct hypotheses; when end_points also holds hyp_sym_R (S,3,3), hyp_sym_t
        (S,3) and hyp_sym_range (B,2) (symmetry.pack_sets), distinct up to each proposal's symmetries"""
        if self.training:
            raise NotImplementedError("sam6d_b200 implements the inference path (model.eval())")
        B = f1.shape[0]
        e = self._embed(_pair(f1, f2))
        f1, f2 = e[:B], e[B:]
        for blk in self.transformers:
            f1, f2 = blk(f1, geo1, f2, geo2)
        S, H = f1.shape[1:]
        w = self._weights()
        o = _gemm(self.precision, _pair(f1, f2).reshape(2 * B * S, H), w["w_out"], w["b_out"]).view(2 * B, S, -1)
        o1, o2 = o[:B], o[B:]
        atten = compute_feature_similarity(o1, o2, self.cfg.sim_type, self.cfg.temp, self.cfg.normalize_feat, self.precision)
        model = ops.scale_by_radius(end_points['model'].contiguous(), radius.contiguous())
        K, min_angle, min_dist = hypotheses
        sym = None
        if K > 1 and all(k in end_points for k in SYM_KEYS):
            sym = tuple(end_points[k].contiguous() for k in SYM_KEYS) + (radius.contiguous(),)
        res = compute_coarse_Rt(atten, p1, p2, model, self.cfg.nproposal1, self.cfg.nproposal2, rand=rand, return_scores=True,
                                n_hypotheses=K, min_angle=min_angle, min_dist=min_dist, symmetries=sym)
        init_R, init_t, self.last_select_scores = res[:3]
        if K > 1:
            end_points['hyp_init_R'], end_points['hyp_init_t'], _, end_points['hyp_valid'], _ = res[3:]
        end_points['init_R'] = init_R
        end_points['init_t'] = init_t
        if self.return_feat:
            return end_points, o1, o2
        return end_points


# =====================================================================================================================
class _ConvBN(nn.Module):
    """pytorch_utils.Conv2d(bn=True): `.conv` (1x1, no bias) + `.normlayer.bn` (PN2/pytorch_utils.py:87-137)"""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size=(1, 1), bias=False)
        self.normlayer = nn.Module()
        self.normlayer.bn = nn.BatchNorm2d(cout)

    def folded(self):
        bn = self.normlayer.bn
        w = self.conv.weight.detach().double().reshape(self.conv.out_channels, -1)
        s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
        return (w * s[:, None]).float().contiguous(), (bn.bias.detach().double() - bn.running_mean.detach().double() * s).float().contiguous()


class _SharedMLP(nn.Module):
    def __init__(self, dims):
        super().__init__()
        for i in range(len(dims) - 1):
            self.add_module(f"layer{i}", _ConvBN(dims[i], dims[i + 1]))


class _Conv1dParams(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv1d(cin, cout, kernel_size=1, bias=True)


class PositionalEncoding(nn.Module):
    """fine_point_matching.py:90-125.  forward(pts (B,N,3)) -> (B,N,out_dim)."""

    def __init__(self, out_dim, r1=0.1, r2=0.2, nsample1=32, nsample2=64, use_xyz=True, bn=True):
        super().__init__()
        if not (use_xyz and bn) or (nsample1, nsample2) != (32, 64):
            raise ValueError("sam6d_b200 PositionalEncoding is built for the SAM-6D configuration")
        self.r1, self.r2, self.ns1, self.ns2 = r1, r2, nsample1, nsample2
        self.mlp1 = _SharedMLP([6, 32, 64, 128])
        self.mlp2 = _SharedMLP([6, 32, 64, 128])
        self.mlp3 = _Conv1dParams(256, out_dim)
        self._packed = _Packed()
        self.precision = "fp32"

    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        w = {}
        for name, mlp in (("m1", self.mlp1), ("m2", self.mlp2)):
            packed = []
            for j in range(3):
                wj, bj = getattr(mlp, f"layer{j}").folded()
                packed += [wj, bj]
            w[name] = tuple(packed)
            w[name + "_tc"] = (packed[0], packed[1], packed[2].to(torch.bfloat16).contiguous(), packed[3],
                               packed[4].to(torch.bfloat16).contiguous(), packed[5])
        w["w3"] = _W(_f32(self.mlp3.conv.weight).reshape(self.mlp3.conv.out_channels, -1))
        w["b3"] = _f32(self.mlp3.conv.bias)
        return w

    @torch.no_grad()
    def local_features(self, pts):
        """the (B,N,256) two-scale max-pooled features before mlp3"""
        w = self._weights()
        pts = pts.contiguous()
        B, N, _ = pts.shape
        feat = torch.empty(B, N, 256, dtype=torch.bfloat16 if self.precision == "bf16" else torch.float32, device=pts.device)
        # ball_query_pair takes the smaller radius first; its outputs are those of two ball_query calls
        (ra, nsa, name_a, off_a), (rb, nsb, name_b, off_b) = sorted(
            ((self.r1, self.ns1, "m1", 0), (self.r2, self.ns2, "m2", 128)), key=lambda s: s[0])
        ia, ca, ib, cb = ops.ball_query_pair(pts, pts, ra, nsa, rb, nsb)
        for name, off, idx, cnt in ((name_a, off_a, ia, ca), (name_b, off_b, ib, cb)):
            if self.precision == "bf16":
                ops.pe_mlp_max_tc(pts, idx, w[name + "_tc"], feat, off)
            else:
                ops.pe_mlp_max(pts, idx, cnt, w[name], feat, off)
        return feat

    @torch.no_grad()
    def forward(self, pts1, pts2=None):
        if pts2 is not None and pts2 is not pts1:
            raise NotImplementedError("SAM-6D always calls PE(pts) with a single cloud")
        w = self._weights()
        feat = self.local_features(pts1)
        B, N, _ = feat.shape
        if self.precision == "bf16":
            return ops.gemm_tma(feat.view(B * N, 256), w["w3"].bf16, w["b3"]).view(B, N, -1)
        return _gemm(self.precision, feat.view(B * N, 256), w["w3"], w["b3"]).view(B, N, -1)


class _LinearAttentionParams(nn.Module):
    def __init__(self, d_model):
        super().__init__()
        self.proj_q = nn.Linear(d_model, d_model)
        self.proj_k = nn.Linear(d_model, d_model)
        self.proj_v = nn.Linear(d_model, d_model)
        self.scale = nn.Parameter(torch.zeros(size=(1, 1, d_model)))


class _LinearAttentionLayerParams(nn.Module):
    def __init__(self, d_model):
        super().__init__()
        self.attention = _LinearAttentionParams(d_model)
        self.linear = nn.Linear(d_model, d_model)
        self.norm = nn.LayerNorm(d_model)


class _LinearTransformerLayerParams(nn.Module):
    def __init__(self, d_model):
        super().__init__()
        self.attention = _LinearAttentionLayerParams(d_model)
        self.output = _AttentionOutputParams(d_model)


class SparseToDenseTransformer(nn.Module):
    """transformer.py:613-673 with with_bg_token=True, replace_bg_token=True (the SAM-6D configuration).
    forward(dense_feats0 (B,N+1,C), embeddings0, fps_idx0, dense_feats1, embeddings1, fps_idx1) -> (dense0, dense1)."""

    def __init__(self, d_model, sparse_blocks, num_heads=4, dropout=None, activation_fn='ReLU', parallel=False,
                 focusing_factor=3, with_bg_token=True, replace_bg_token=True):
        super().__init__()
        if not (with_bg_token and replace_bg_token) or focusing_factor != 3:
            raise ValueError("sam6d_b200 SparseToDenseTransformer is built for the SAM-6D configuration")
        self.d_model = d_model
        self.sparse_layer = GeometricTransformer(blocks=sparse_blocks, d_model=d_model, num_heads=num_heads, dropout=dropout,
                                                 activation_fn=activation_fn, parallel=parallel, return_attention_scores=False)
        self.dense_layer = _LinearTransformerLayerParams(d_model)
        self._packed = _Packed()
        self.precision = "fp32"

    def _weights(self):
        return self._packed.get(self._pack, self.dense_layer)

    def _pack(self):
        la = self.dense_layer.attention.attention
        return dict(
            wq=_W(la.proj_q.weight), bq=_f32(la.proj_q.bias),
            wkv=_W(torch.cat([_f32(la.proj_k.weight), _f32(la.proj_v.weight)], dim=0)),
            bkv=torch.cat([_f32(la.proj_k.bias), _f32(la.proj_v.bias)], dim=0).contiguous(),
            sp_scale=torch.nn.functional.softplus(_f32(la.scale)).reshape(-1).contiguous(), tail=_pack_tail(self.dense_layer))

    def _sample_feats(self, dense_feats, idx_ext):
        # quirk Q1 (transformer.py:651-658): the gather runs on the bg-prefixed sequence with the raw FPS index
        if dense_feats.dtype == torch.bfloat16:
            return ops.gather_rows_bf16(dense_feats, idx_ext)
        return ops.gather_rows(dense_feats, idx_ext)

    def _dense_layer_bf16(self, dense, sparse, w):
        """_dense_layer for the bf16 token stream: dense (B,N+1,C) bf16, sparse (B,J+1,C) bf16.  Every GEMM is the persistent
        TMA kernel over all B*(N+1) rows (the bg row rides along and is overwritten at the end), the feature map and the
        per-head (q' KV) / (q' . ksum) run in one wgmma kernel, LayerNorms read and write bf16."""
        B, N1, C = dense.shape
        N, J = N1 - 1, sparse.shape[1] - 1
        dev = dense.device
        bf = torch.bfloat16
        x2d = dense.view(B * N1, C)
        q = ops.gemm_tma(x2d, w["wq"].bf16, w["bq"], out_dtype=bf)
        kv = torch.empty(B * J, 2 * C, dtype=torch.float32, device=dev)
        ops.gemm_tc(sparse[:, 1:, :], w["wkv"].bf16, w["bkv"], out=kv.view(B, J, 2 * C))
        ops.focus_rows(kv[:, :C], w["sp_scale"], out=kv[:, :C])
        kv3 = kv.view(B, J, 2 * C)
        blob, KS = ops.linattn_kv_pack(kv3[..., :C], kv3[..., C:])
        x_att = torch.empty(B * N1, C, dtype=bf, device=dev)
        ops.linattn_tc(q.view(B, N1, C)[:, 1:, :], blob, KS, w["sp_scale"], x_att.view(B, N1, C)[:, 1:, :])
        x_att.view(B, N1, C)[:, 0, :] = 0                                   # bg rows: defined input for the tail below
        out = _tail_bf16(x2d, x_att, w["tail"]).view(B, N1, C)
        out[:, 0, :] = sparse[:, 0, :].to(bf)                               # replaced bg token (transformer.py:660-668)
        return out

    def _dense_layer(self, dense, sparse, w):
        """LinearTransformerLayer on dense[:,1:,:] with memory sparse[:,1:,:]; returns the new (B,N+1,C) sequence."""
        B, N1, C = dense.shape
        N, J = N1 - 1, sparse.shape[1] - 1
        dev = dense.device
        x = dense[:, 1:, :]                                                 # rows 1..N of every proposal
        q = torch.empty(B * N, C, dtype=torch.float32, device=dev)
        prec = self.precision
        _gemm(prec, x, w["wq"], w["bq"], out=q.view(B, N, C))
        kv = torch.empty(B * J, 2 * C, dtype=torch.float32, device=dev)
        _gemm(prec, sparse[:, 1:, :], w["wkv"], w["bkv"], out=kv.view(B, J, 2 * C))
        ops.focus_rows(q, w["sp_scale"], out=q)
        ops.focus_rows(kv[:, :C], w["sp_scale"], out=kv[:, :C])
        KV = torch.empty(B, NUM_HEADS, 64, 64, dtype=torch.float32, device=dev)
        KS = torch.empty(B, NUM_HEADS, 64, dtype=torch.float32, device=dev)
        kv3 = kv.view(B, J, 2 * C)
        ops.linattn_kv(kv3[..., :C], kv3[..., C:], KV, KS)
        x_att = torch.empty(B * N, C, dtype=torch.float32, device=dev)
        ops.linattn_apply(q.view(B, N, C), KV, KS, x_att.view(B, N, C))
        t = w["tail"]
        y = torch.empty(B * N, C, dtype=torch.float32, device=dev)
        _gemm(prec, x_att.view(B, N, C), t["wo"], t["bo"], residual=x, out=y.view(B, N, C))
        y = ops.layernorm(y, t["g1"], t["b1"])
        h = _gemm(prec, y, t["we"], t["be"], relu=True)
        z = _gemm(prec, h, t["ws"], t["bs"], residual=y)
        out = torch.empty(B, N1, C, dtype=torch.float32, device=dev)
        ops.layernorm(z, t["g2"], t["b2"], out=out[:, 1:, :])
        out[:, 0, :] = sparse[:, 0, :]                                      # replaced bg token (transformer.py:660-668)
        return out

    @torch.no_grad()
    def forward(self, dense_feats0, embeddings0, fps_idx0, dense_feats1, embeddings1, fps_idx1, masks0=None, masks1=None):
        w = self._weights()
        B = dense_feats0.shape[0]
        idx = torch.cat([fps_idx0, fps_idx1], dim=0)
        ext = torch.cat([torch.zeros_like(idx[:, :1]), idx], dim=1)
        layer = self._dense_layer_bf16 if dense_feats0.dtype == torch.bfloat16 else self._dense_layer
        stacked = dense_feats0.shape == dense_feats1.shape
        if stacked:
            # one batch of 2B clouds through the gather, the (shared-weight) dense linear-attention layer and its FFN
            dense = _pair(dense_feats0, dense_feats1)
            feats = self._sample_feats(dense, ext)
        else:
            # unequal point counts: the gather and the dense layer run per cloud; the sparse clouds have equal sizes
            feats = torch.cat([self._sample_feats(dense_feats0.contiguous(), ext[:B]),
                               self._sample_feats(dense_feats1.contiguous(), ext[B:])])
        feats0, feats1 = self.sparse_layer(feats[:B], embeddings0, feats[B:], embeddings1, masks0, masks1)
        if not stacked:
            return layer(dense_feats0.contiguous(), feats0, w), layer(dense_feats1.contiguous(), feats1, w)
        out = layer(dense, _pair(feats0, feats1), w)
        return out[:B], out[B:]


class FinePointMatching(nn.Module):
    """forward(p1, f1, geo1, fps_idx1, p2, f2, geo2, fps_idx2, radius, end_points) -> end_points with pred_R/pred_t/pred_pose_score."""

    def __init__(self, cfg, return_feat=False):
        super().__init__()
        self.cfg = _cfg(cfg)
        self.return_feat = return_feat
        self.nblock = self.cfg.nblock
        self.in_proj = nn.Linear(self.cfg.input_dim, self.cfg.hidden_dim)
        self.out_proj = nn.Linear(self.cfg.hidden_dim, self.cfg.out_dim)
        self.bg_token = nn.Parameter(torch.randn(1, 1, self.cfg.hidden_dim) * .02)
        self.PE = PositionalEncoding(self.cfg.hidden_dim, r1=self.cfg.pe_radius1, r2=self.cfg.pe_radius2)
        self._packed = _Packed()
        self.precision = "fp32"
        self.transformers = nn.ModuleList([
            SparseToDenseTransformer(self.cfg.hidden_dim, num_heads=4, sparse_blocks=['self', 'cross'], dropout=None,
                                     activation_fn='ReLU', focusing_factor=self.cfg.focusing_factor, with_bg_token=True,
                                     replace_bg_token=True) for _ in range(self.nblock)])

    def _weights(self):
        return self._packed.get(lambda: dict(w_in=_W(self.in_proj.weight), b_in=_f32(self.in_proj.bias), w_out=_W(self.out_proj.weight),
                                             b_out=_f32(self.out_proj.bias)), self.in_proj, self.out_proj)

    def _embed(self, f, pts):
        """[bg_token ; in_proj(f) + PE(pts)] as one (B,N+1,H) sequence (fine_point_matching.py:46-50)"""
        B, N, C = f.shape
        H = self.cfg.hidden_dim
        w, pw = self._weights(), self.PE._weights()
        local = self.PE.local_features(pts)                                         # (B,N,256)
        if self.precision == "bf16":
            # the dense token stream of the fine stage is bf16 from here on (fp32 accumulation inside every kernel):
            # in_proj(f) in bf16 is the residual of the mlp3 GEMM over the bf16 local features, written behind the bg row
            f2d = f.reshape(B * N, C)
            if f2d.dtype == torch.bfloat16 and f2d.is_contiguous():
                tmp = ops.gemm_tma(f2d, w["w_in"].bf16, w["b_in"], out_dtype=torch.bfloat16)
            else:
                tmp = ops.gemm_tc(f2d, w["w_in"].bf16, w["b_in"], out_dtype=torch.bfloat16)
            out = torch.empty(B, N + 1, H, dtype=torch.bfloat16, device=f.device)
            out[:, 0, :] = self.bg_token.detach().reshape(1, -1).to(torch.bfloat16)
            ops.gemm_tma_batched(local, pw["w3"].bf16, out[:, 1:, :], bias=pw["b3"], residual=tmp.view(B, N, H))
            return out
        tmp = _gemm(self.precision, f.reshape(B * N, C), w["w_in"], w["b_in"])
        out = torch.empty(B, N + 1, H, dtype=torch.float32, device=f.device)
        out[:, 0, :] = self.bg_token.detach().reshape(1, -1)
        _gemm(self.precision, local, pw["w3"], pw["b3"], residual=tmp.view(B, N, H), out=out[:, 1:, :])
        return out

    @torch.no_grad()
    def forward(self, p1, f1, geo1, fps_idx1, p2, f2, geo2, fps_idx2, radius, end_points):
        if self.training:
            raise NotImplementedError("sam6d_b200 implements the inference path (model.eval())")
        p1, p2 = p1.contiguous(), p2.contiguous()
        p1_ = ops.rigid_warp(p1, end_points['init_R'].contiguous(), end_points['init_t'].contiguous())
        if p1.shape == p2.shape:
            e = self._embed(_pair(f1, f2), torch.cat([p1_, p2], dim=0))    # both clouds: one PE pass, one in_proj GEMM
            f1, f2 = e[:p1.shape[0]], e[p1.shape[0]:]
        else:
            f1 = self._embed(f1.contiguous(), p1_)
            f2 = self._embed(f2.contiguous(), p2)
        for blk in self.transformers:
            f1, f2 = blk(f1, geo1, fps_idx1, f2, geo2, fps_idx2)
        B, S, H = f1.shape
        w = self._weights()
        if f1.shape == f2.shape:
            o = _gemm(self.precision, _pair(f1, f2).reshape(2 * B * S, H), w["w_out"], w["b_out"]).view(2 * B, S, -1)
            o1, o2 = o[:B], o[B:]
        else:
            o1 = _gemm(self.precision, f1.reshape(B * S, H), w["w_out"], w["b_out"]).view(B, S, -1)
            o2 = _gemm(self.precision, f2.reshape(B * S, H), w["w_out"], w["b_out"]).view(B, S, -1)
        model = ops.scale_by_radius(end_points['model'].contiguous(), radius.contiguous())
        if (self.precision == "bf16" and self.cfg.sim_type == 'cosine' and self.cfg.normalize_feat and H == 256
                and o1.shape[-1] == 256 and not self.return_feat):
            # score tiles are recomputed on the tensor cores inside every assignment pass: no (B,2049,2049) matrix in HBM
            f1n, f2n = ops.l2norm_rows_bf16(o1.contiguous()), ops.l2norm_rows_bf16(o2.contiguous())
            lab1, _, wts, pred = ops.fine_assign_tc(f1n, f2n, p2, 1.0 / self.cfg.temp)
            pred_R, pred_t = ops.weighted_procrustes(pred, p1, wts, 0.0, 1e-5)
            score, t_scaled = ops.pose_score(p1, lab1, pred_R, pred_t, model.contiguous(), radius.contiguous(), 0.15)
        else:
            if not self.cfg.normalize_feat:
                raise NotImplementedError("FinePointMatching: normalize_feat=False scores are unbounded; the fixed-shift assignment "
                                          "kernels need cosine similarities (the SAM-6D configuration)")
            atten = compute_feature_similarity(o1, o2, self.cfg.sim_type, self.cfg.temp, self.cfg.normalize_feat, self.precision)
            # cosine scores of normalised features: bounded by 1/temp by construction, no read-back (keeps the forward capturable)
            pred_R, _, score, t_scaled = compute_fine_Rt(atten, p1, p2, model, temp=self.cfg.temp, radius=radius.contiguous(),
                                                         check_bound=False)
        end_points['pred_R'] = pred_R
        end_points['pred_t'] = t_scaled
        end_points['pred_pose_score'] = score
        if self.return_feat:
            return end_points, o1, o2
        return end_points


# =====================================================================================================================
DEFAULT_MODEL_CFG = dict(
    coarse_npoint=196, fine_npoint=2048,
    geo_embedding=dict(sigma_d=0.2, sigma_a=15, angle_k=3, reduction_a='max', hidden_dim=256),
    coarse_point_matching=dict(nblock=3, input_dim=256, hidden_dim=256, out_dim=256, temp=0.1, sim_type='cosine',
                               normalize_feat=True, loss_dis_thres=0.15, nproposal1=6000, nproposal2=300),
    fine_point_matching=dict(nblock=3, input_dim=256, hidden_dim=256, out_dim=256, pe_radius1=0.1, pe_radius2=0.2,
                             focusing_factor=3, temp=0.1, sim_type='cosine', normalize_feat=True, loss_dis_thres=0.15),
)  # PEM/config/base.yaml:17-54

MAX_HYPOTHESES = 16            # Net.set_hypotheses: fine-stage passes per forward
# the outputs a forward with K > 1 hypotheses adds (Net.set_hypotheses), as graph.StepGraphs copies them out of a replay
HYP_KEYS = ("hyp_init_R", "hyp_init_t", "hyp_R", "hyp_t", "hyp_pose_score", "hyp_valid", "hyp_index")
# inputs that make the K > 1 pick distinct up to the objects' symmetries (symmetry.pack_sets; CoarsePointMatching.forward)
SYM_KEYS = ("hyp_sym_R", "hyp_sym_t", "hyp_sym_range")


def check_hypotheses(k, min_angle, min_dist):
    """-> (k, min_angle, min_dist) as int, float, float; ValueError unless 1 <= k <= MAX_HYPOTHESES, 0 < min_angle <= 180
    (degrees) and min_dist >= 0, both finite"""
    if isinstance(k, bool) or int(k) != k or not 1 <= int(k) <= MAX_HYPOTHESES:
        raise ValueError(f"the number of hypotheses must be an integer in [1, {MAX_HYPOTHESES}], got {k}")
    if not (math.isfinite(min_angle) and 0.0 < min_angle <= 180.0):
        raise ValueError(f"min_angle must lie in (0, 180] degrees, got {min_angle}")
    if not (math.isfinite(min_dist) and min_dist >= 0.0):
        raise ValueError(f"min_dist must be a finite number >= 0, got {min_dist}")
    return int(k), float(min_angle), float(min_dist)


def first_best(score: torch.Tensor, valid: torch.Tensor) -> torch.Tensor:
    """(B,K) scores and valid flags -> (B) i64 the first k with the largest score among the valid slots; a NaN score never
    wins, and a row with nothing to choose gives 0"""
    ok = valid.bool() & ~torch.isnan(score)
    return torch.where(ok, score, torch.full_like(score, -math.inf)).argmax(dim=1)


class Net(nn.Module):
    """Pose_Estimation_Model `Net` (pose_estimation_model.py:11-53).

    forward(end_points) consumes the reference's dict -- 'pts' (B,N,3), 'rgb', 'rgb_choose', 'model' (B,Nm,3), 'dense_po',
    'dense_fo' -- and adds init_R, init_t, pred_R, pred_t, pred_pose_score.  The RGB backbone (`feature_extraction`, a timm
    ViT-B in the reference; SURVEY.md 8f row N1) is pluggable: pass any module with the reference's ViTEncoder interface as
    `feature_extraction`, or put the per-point features into end_points['dense_fm'] (B,N,256) directly.
    """

    def __init__(self, cfg=None, feature_extraction: Optional[nn.Module] = None, precision: str = "fp32"):
        super().__init__()
        cfg = _cfg(cfg if cfg is not None else DEFAULT_MODEL_CFG)
        self.cfg = cfg
        self.coarse_npoint = cfg.coarse_npoint
        self.fine_npoint = cfg.fine_npoint
        if feature_extraction is not None:
            self.feature_extraction = feature_extraction
        elif hasattr(cfg, "feature_extraction"):
            # `Net(cfg.model)` of the reference (PEM/config/base.yaml:18-24): the ViT-B RGB branch under the reference's module
            # name, so that sam-6d-pem-base.pth loads strict=True and model.feature_extraction.get_obj_feats exists
            from .vit import ViTEncoder
            self.feature_extraction = ViTEncoder(cfg.feature_extraction, cfg.fine_npoint, precision)
        self.geo_embedding = GeometricStructureEmbedding(cfg.geo_embedding)
        self.coarse_point_matching = CoarsePointMatching(cfg.coarse_point_matching)
        self.fine_point_matching = FinePointMatching(cfg.fine_point_matching)
        self._graphs = None
        self.hypotheses = (1, 30.0, 0.2)
        self.set_precision(precision)

    def enable_graphs(self, max_graphs: int = 8):
        """replay repeated fixed-shape calls of forward() as one CUDA graph each (sam6d_b200/graph.py: a call signature seen for
        the second time is captured, reading the caller's tensors in place; results are identical to the launch-by-launch
        forward, which stays the path for first sightings, `init_pose` calls and `disable_graphs()`)"""
        from .graph import StepGraphs
        self._graphs = StepGraphs(max_graphs)
        return self

    def disable_graphs(self):
        self._graphs = None
        return self

    def set_precision(self, precision: str):
        """'fp32' (CUDA-core kernels, exact path) or 'bf16' (wgmma tensor-core kernels, bf16 operands / fp32 accumulate)"""
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}")
        self.precision = precision
        for m in self.modules():
            if hasattr(m, "precision") and m is not self:
                m.precision = precision
        return self

    def set_hypotheses(self, k: int = 1, min_angle: float = 30.0, min_dist: float = 0.2):
        """run the fine stage from k mutually distinct coarse hypotheses and keep the best (not in the reference).  Two
        hypotheses are distinct when their rotations differ by at least min_angle degrees or their translations by at least
        min_dist object radii (ops.coarse_pick_distinct).  forward() then runs the coarse stage once and the fine stage once per
        hypothesis on the same batch, and reports, per proposal, the pass with the largest pred_pose_score among the valid
        ones (the first on a tie), plus hyp_init_R (B,k,3,3), hyp_init_t (B,k,3), hyp_R, hyp_t, hyp_pose_score (B,k), hyp_valid
        (B,k) u8 and hyp_index (B) i64; init_R and init_t stay the coarse stage's pick.  k = 1 (default): the reference's
        forward, with no hyp_* output."""
        self.hypotheses = check_hypotheses(k, min_angle, min_dist)
        return self

    def _features(self, end_points):
        """ViTEncoder.forward, inference branch (feature_extraction.py:128-142)"""
        if 'dense_fm' in end_points:
            dense_fm = end_points['dense_fm']
        elif hasattr(self, 'feature_extraction'):
            dense_fm = self.feature_extraction.get_img_feats(end_points['rgb'], end_points['rgb_choose'])
        else:
            raise RuntimeError("Net needs end_points['dense_fm'] or a feature_extraction module for the RGB branch")
        if 'dense_po' not in end_points or 'dense_fo' not in end_points:
            raise RuntimeError("inference needs the template bank: end_points['dense_po'], end_points['dense_fo']")
        dense_po = end_points['dense_po'].contiguous()
        radius = ops.cloud_radius(dense_po)
        dense_pm = ops.scale_by_radius(end_points['pts'].contiguous(), radius)
        dense_po = ops.scale_by_radius(dense_po, radius)
        return dense_pm, dense_fm.contiguous(), dense_po, end_points['dense_fo'].contiguous(), radius

    @torch.no_grad()
    def forward(self, end_points, rand=None, init_pose=None):
        """rand: the (B, 3*nproposal1) uniforms of compute_coarse_Rt (default: drawn like the reference).  init_pose = (R, t):
        the fine stage starts from this pose instead of the coarse stage's (the coarse stage still runs and reports init_R /
        init_t); used by the parity tests to hold the fine stage to the 1e-3 bar independently of the coarse stage's discrete
        hypothesis selection.  A call with init_pose runs one fine pass whatever set_hypotheses chose."""
        if self.training:
            raise NotImplementedError("sam6d_b200 implements the inference path: call model.eval()")
        if self._graphs is not None and init_pose is None and 'pts' in end_points:
            n_rand = self.coarse_point_matching.cfg.nproposal1 * 3
            out = self._graphs.run(lambda ep, r: self._forward(ep, r, None), end_points, rand, n_rand,
                                   extra=(self.precision, hash(_param_key(self)), self.hypotheses),
                                   keys=HYP_KEYS if self.hypotheses[0] > 1 else ())
            if out is not None:
                return out
        return self._forward(end_points, rand, init_pose)

    def _forward(self, end_points, rand, init_pose):
        dense_pm, dense_fm, dense_po, dense_fo, radius = self._features(end_points)
        B = dense_pm.size(0)
        if dense_pm.shape == dense_po.shape and dense_fm.shape == dense_fo.shape:
            # Scene and template clouds share every weight up to the cross-attention, so they travel as the two halves of
            # one (2B, ...) allocation: FPS, the geometric embedding, PE, the self-attention and dense layers each run once
            # on 2B clouds; the views below keep the reference's two-argument interfaces.
            pts2 = torch.cat([dense_pm, dense_po], dim=0)
            if self.precision == "bf16":
                # every consumer of the point features rounds them to bf16 operands (in_proj of both stages): round once while
                # stacking -- 134 MB read + 67 MB written instead of a 268 MB fp32 copy, and the fine in_proj reads 67 MB by TMA
                fts2 = torch.empty(2 * B, *dense_fm.shape[1:], dtype=torch.bfloat16, device=dense_fm.device)
                fts2[:B].copy_(dense_fm)
                fts2[B:].copy_(dense_fo)
            else:
                fts2 = torch.cat([dense_fm, dense_fo], dim=0)
            dense_pm, dense_po, dense_fm, dense_fo = pts2[:B], pts2[B:], fts2[:B], fts2[B:]
            sp, sf, idx = sample_pts_feats(pts2, fts2, self.coarse_npoint, return_index=True)
        else:
            # unequal point counts: FPS, PE and the dense layers run per cloud; both clouds come down to coarse_npoint points,
            # so the geometric embedding and the sparse stage still run on 2B clouds
            m = sample_pts_feats(dense_pm, dense_fm, self.coarse_npoint, return_index=True)
            o = sample_pts_feats(dense_po, dense_fo, self.coarse_npoint, return_index=True)
            sp, sf, idx = (torch.cat(z) for z in zip(m, o))
        bg_point = torch.ones(2 * B, 1, 3, dtype=torch.float32, device=sp.device) * 100
        geo = self.geo_embedding(torch.cat([bg_point, sp], dim=1))
        sparse_pm, sparse_po, sparse_fm, sparse_fo = sp[:B], sp[B:], sf[:B], sf[B:]
        fps_idx_m, fps_idx_o, geo_embedding_m, geo_embedding_o = idx[:B], idx[B:], geo[:B], geo[B:]
        K = self.hypotheses[0] if init_pose is None else 1
        end_points = self.coarse_point_matching(sparse_pm, sparse_fm, geo_embedding_m, sparse_po, sparse_fo, geo_embedding_o,
                                                radius, end_points, rand=rand, hypotheses=(K,) + self.hypotheses[1:])
        if K > 1:
            # one fine pass per hypothesis over the same B proposals: every pass reuses the clouds, features and geometric
            # embeddings above (a (B K)-batch would copy the ~20 MB per-cloud embedding K times)
            passes = []
            for k in range(K):
                ep = dict(end_points, init_R=end_points['hyp_init_R'][:, k].contiguous(),
                          init_t=end_points['hyp_init_t'][:, k].contiguous())
                ep = self.fine_point_matching(dense_pm, dense_fm, geo_embedding_m, fps_idx_m, dense_po, dense_fo, geo_embedding_o,
                                              fps_idx_o, radius, ep)
                passes.append((ep['pred_R'], ep['pred_t'], ep['pred_pose_score']))
            hyp_R, hyp_t, hyp_s = (torch.stack(z, dim=1) for z in zip(*passes))
            idx = first_best(hyp_s, end_points['hyp_valid'])
            rows = torch.arange(B, device=idx.device)
            end_points.update(hyp_R=hyp_R, hyp_t=hyp_t, hyp_pose_score=hyp_s, hyp_index=idx, pred_R=hyp_R[rows, idx],
                              pred_t=hyp_t[rows, idx], pred_pose_score=hyp_s[rows, idx])
            return end_points
        if init_pose is not None:
            coarse_R, coarse_t = end_points['init_R'], end_points['init_t']
            end_points['init_R'], end_points['init_t'] = init_pose[0].contiguous(), init_pose[1].contiguous()
        end_points = self.fine_point_matching(dense_pm, dense_fm, geo_embedding_m, fps_idx_m, dense_po, dense_fo,
                                              geo_embedding_o, fps_idx_o, radius, end_points)
        if init_pose is not None:
            end_points['init_R'], end_points['init_t'] = coarse_R, coarse_t
        return end_points
