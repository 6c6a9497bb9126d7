"""CPU: the float64 restatements of tests/_fp32_ref.py against oracle/pem_oracle.py and the torch functional forms.  The GPU
bounds of tests/test_gpu_fp32_kernels.py are only as good as these restatements: each is composed here into the oracle's layer
(RPE self-attention, cross-attention, linear attention, geometric embedding, positional encoding) and must agree with it."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp32_ref as R   # noqa: E402
from oracle import pem_oracle as po   # noqa: E402

F64 = torch.float64


@pytest.fixture(scope="module")
def sd64():
    return {k: (v.double() if v.is_floating_point() else v) for k, v in po.make_state_dict(seed=3).items()}


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b, rtol):
    err = (a - b).abs().max().item()
    scale = b.abs().max().item()
    assert err <= rtol * scale, f"max |diff| {err:.3g} > {rtol:g} x max |ref| {scale:.3g}"


def _tail(sd, p, x2d, hid):
    """attention.linear + residual, attention.norm, then AttentionOutput, all through the restatements"""
    y, _ = R.gemm(hid, sd[p + ".attention.linear.weight"], sd[p + ".attention.linear.bias"], residual=x2d)
    y, _ = R.layernorm(y, sd[p + ".attention.norm.weight"], sd[p + ".attention.norm.bias"], 1e-5)
    h, _ = R.gemm(y, sd[p + ".output.expand.weight"], sd[p + ".output.expand.bias"], act=1)
    z, _ = R.gemm(h, sd[p + ".output.squeeze.weight"], sd[p + ".output.squeeze.bias"], residual=y)
    return R.layernorm(z, sd[p + ".output.norm.weight"], sd[p + ".output.norm.bias"], 1e-5)[0]


def test_rpe_self_layer_matches_oracle(sd64):
    """qkvu projection with proj_p folded into the query as sam6d_b200.pem folds it, rpe_scores, mha and the tail"""
    B, S, C = 2, 37, 256
    g = _g(0)
    x = torch.randn(B, S, C, generator=g, dtype=F64)
    emb = torch.randn(B, S, S, C, generator=g, dtype=F64)
    p = "coarse_point_matching.transformers.0.layers.0"
    a = p + ".attention.attention"
    wq, bq, wp = sd64[a + ".proj_q.weight"], sd64[a + ".proj_q.bias"], sd64[a + ".proj_p.weight"]
    mu = [wp[h * 64:(h + 1) * 64].t() @ wq[h * 64:(h + 1) * 64] for h in range(4)]
    cu = [wp[h * 64:(h + 1) * 64].t() @ bq[h * 64:(h + 1) * 64] for h in range(4)]
    w_self = torch.cat([wq, sd64[a + ".proj_k.weight"], sd64[a + ".proj_v.weight"]] + mu)
    b_self = torch.cat([bq, sd64[a + ".proj_k.bias"], sd64[a + ".proj_v.bias"]] + cu)
    x2d = x.reshape(B * S, C)
    qkvu, _ = R.gemm(x2d, w_self, b_self)
    sp, _ = R.rpe_scores(emb, qkvu[:, 3 * C:])
    qkv = qkvu.view(B, S, -1)
    hid, _ = R.mha(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:3 * C], sp, 1.0 / 8.0)
    got = _tail(sd64, p, x2d, hid.reshape(B * S, C)).view(B, S, C)
    _close(got, po.rpe_self_layer(sd64, p, x, emb), 1e-10)


def test_cross_layer_matches_oracle(sd64):
    B, S, Sm, C = 2, 29, 41, 256
    g = _g(1)
    x = torch.randn(B, S, C, generator=g, dtype=F64)
    mem = torch.randn(B, Sm, C, generator=g, dtype=F64)
    p = "coarse_point_matching.transformers.0.layers.1"
    a = p + ".attention.attention"
    q, _ = R.gemm(x.reshape(B * S, C), sd64[a + ".proj_q.weight"], sd64[a + ".proj_q.bias"])
    k, _ = R.gemm(mem.reshape(B * Sm, C), sd64[a + ".proj_k.weight"], sd64[a + ".proj_k.bias"])
    v, _ = R.gemm(mem.reshape(B * Sm, C), sd64[a + ".proj_v.weight"], sd64[a + ".proj_v.bias"])
    hid, _ = R.mha(q.view(B, S, C), k.view(B, Sm, C), v.view(B, Sm, C), None, 1.0 / 8.0)
    got = _tail(sd64, p, x.reshape(B * S, C), hid.reshape(B * S, C)).view(B, S, C)
    _close(got, po.cross_layer(sd64, p, x, mem), 1e-10)


@pytest.mark.parametrize("N,J", [(300, 40), (5, 60)])
def test_linear_attention_matches_oracle(sd64, N, J):
    """focus_rows on q and k, linattn_kv, linattn_apply; (5, 60) takes the oracle's qk-first branch"""
    B, C = 2, 256
    g = _g(2)
    xq = torch.randn(B, N, C, generator=g, dtype=F64)
    xkv = torch.randn(B, J, C, generator=g, dtype=F64)
    p = "fine_point_matching.transformers.0.dense_layer.attention.attention"
    sd = dict(sd64)
    sd[p + ".scale"] = 0.3 * torch.randn(1, 1, C, generator=g, dtype=F64)     # away from the zero initialisation
    q, _ = R.gemm(xq, sd[p + ".proj_q.weight"], sd[p + ".proj_q.bias"])
    k, _ = R.gemm(xkv, sd[p + ".proj_k.weight"], sd[p + ".proj_k.bias"])
    v, _ = R.gemm(xkv, sd[p + ".proj_v.weight"], sd[p + ".proj_v.bias"])
    sp = F.softplus(sd[p + ".scale"]).reshape(-1)
    fq, _ = R.focus(q.reshape(-1, C), sp)
    fk, _ = R.focus(k.reshape(-1, C), sp)
    KV, KS, _, _ = R.linattn_kv(fk.view(B, J, C), v)
    got, _ = R.linattn_apply(fq.view(B, N, C), KV, KS)
    _close(got, po.linear_attention(sd, p, xq, xkv), 1e-9)


def test_geo_embedding_matches_oracle(sd64):
    B, S = 2, 23
    pts = torch.randn(B, S, 3, generator=_g(4), dtype=F64) * 0.1
    pts[:, 0] = 100.0                                   # a far point: distance indices near 866 in its row and column
    d_idx, a_idx = po.geo_embedding_indices(pts)
    T = torch.cat([a_idx, d_idx.unsqueeze(-1)], -1).reshape(-1, 4)
    pre = "geo_embedding"
    div = torch.exp(torch.arange(0, 256, 2).float() * (-math.log(10000.0) / 256))
    assert torch.equal(div.double(), sd64[pre + ".embedding.div_term"])
    x = torch.linspace(0, 900, 77, dtype=F64)
    _close(R.sin_emb(x, div, arg_fp32=False), po.sinusoidal_embedding(x, 256), 1e-15)
    E, _ = R.geo_embed(T, div, sd64[pre + ".proj_a.weight"].t(), sd64[pre + ".proj_d.weight"].t(),
                       sd64[pre + ".proj_a.bias"] + sd64[pre + ".proj_d.bias"], arg_fp32=False)
    _close(E.view(B, S, S, 256), po.geo_embedding(sd64, pts), 1e-12)


def test_geo_argument_rounding_is_within_its_size():
    """with fp32 indices the restatement forms x * div_term[f] in fp32, as the kernel does: it moves each sin / cos by at most
    |x w| u, so its difference to the float64 argument stays within that (and is not zero at the large indices)"""
    div = torch.exp(torch.arange(0, 256, 2).float() * (-math.log(10000.0) / 256))
    x = torch.linspace(0, 900, 301).float()
    a, b = R.sin_emb(x, div, arg_fp32=True), R.sin_emb(x.double(), div, arg_fp32=False)
    lim = (x.double().unsqueeze(-1) * div.double()).repeat_interleave(2, -1) * R.U
    assert ((a - b).abs() <= lim * 1.0001 + 1e-300).all()
    assert (a - b).abs().max() > 0


def test_positional_encoding_matches_oracle(sd64):
    """the PE SharedMLPs with BatchNorm folded as sam6d_b200.pem folds them, the ball-query count read off the padded index
    list, the max over samples, then mlp3 -- against the oracle in fp32 (its ball query runs on fp32 points)"""
    from sam6d_b200.pem import _ConvBN
    from oracle import pn2
    B, N = 2, 300
    pts = (torch.rand(B, N, 3, generator=_g(5)) - 0.5) * 0.3
    pre = "fine_point_matching.PE"
    sd32 = {k: (v.float() if v.is_floating_point() else v) for k, v in sd64.items()}
    feats = []
    for name, r, ns in (("mlp1", po.PE_R1, po.PE_NS1), ("mlp2", po.PE_R2, po.PE_NS2)):
        idx = pn2.ball_query(pts, pts, r, ns)
        cnt = (idx[..., 1:] > idx[..., :-1]).int().cumprod(-1).sum(-1) + 1      # found indices ascend; padding repeats idx[0]
        assert (cnt < ns).any() and (cnt == ns).any()
        w = []
        for j in range(3):
            m = _ConvBN(*sd32[f"{pre}.{name}.layer{j}.conv.weight"].shape[1::-1])
            m.load_state_dict({k[len(f"{pre}.{name}.layer{j}."):]: v for k, v in sd32.items()
                               if k.startswith(f"{pre}.{name}.layer{j}.")})
            wj, bj = m.eval().folded()
            ref_w, ref_b = R.fold_bn(sd64[f"{pre}.{name}.layer{j}.conv.weight"], *(sd64[f"{pre}.{name}.layer{j}.normlayer.bn.{s}"]
                                     for s in ("weight", "bias", "running_mean", "running_var")))
            assert torch.allclose(wj.double(), ref_w, rtol=1e-6, atol=1e-7)
            w += [wj, bj]
        feats.append(R.pe_mlp_max(pts, idx, cnt, w)[0])
    feat = torch.cat(feats, -1)
    got, _ = R.gemm(feat, sd64[pre + ".mlp3.conv.weight"].reshape(256, 256), sd64[pre + ".mlp3.conv.bias"])
    _close(got, po.positional_encoding(sd32, pts).double(), 2e-5)


def test_row_ops_match_torch():
    g = _g(6)
    for C in (32, 256, 1536):
        x = torch.randn(40, C, generator=g, dtype=F64) * 3 + 2
        gm, bt = torch.randn(C, generator=g, dtype=F64), torch.randn(C, generator=g, dtype=F64)
        for eps in (1e-5, 1e-6):
            _close(R.layernorm(x, gm, bt, eps)[0], F.layer_norm(x, (C,), gm, bt, eps), 1e-14)
        x[3] = 0
        x[4] *= 1e-14                                   # norm below the clamp: differs from F.normalize's 1e-12 by 4e-9
        _close(R.l2norm(x)[0], F.normalize(x, dim=-1, eps=1e-12), 1e-8)
    z = torch.linspace(-8, 8, 1001, dtype=F64)
    _close(R.gelu(z), F.gelu(z, approximate="none"), 1e-7)        # the fp32 constant 0.70710678f, not 1/sqrt(2)
    y, e = R.gemm(z.view(-1, 1), torch.ones(1, 1, dtype=F64), act=2)
    assert torch.equal(y.view(-1), R.gelu(z)) and (e > 0).all()


def test_point_ops_match_direct_forms():
    g = _g(7)
    p = torch.randn(3, 50, 3, generator=g, dtype=F64)
    Rm = torch.linalg.qr(torch.randn(3, 3, 3, generator=g, dtype=F64))[0]
    t = torch.randn(3, 3, generator=g, dtype=F64)
    out, _ = R.rigid_warp(p, Rm, t)
    _close(out, torch.einsum("bnk,bkj->bnj", p - t[:, None], Rm), 1e-15)
    r, _ = R.cloud_radius(p)
    assert torch.allclose(r, torch.tensor([max(v.norm().item() for v in c) for c in p], dtype=F64), rtol=1e-15)
    s, _ = R.scale_by_radius(p, r)
    _close(s, p / (r.view(-1, 1, 1) + R.EPS6), 1e-15)


def test_bounds_reject_wrong_answers_on_paper():
    """the negative controls the GPU file uses move the answer by more than the bound on operands where the bound is tight"""
    g = _g(8)
    x = torch.randn(64, 256, generator=g, dtype=F64)
    ok, e = R.layernorm(x, torch.ones(256, dtype=F64), torch.zeros(256, dtype=F64), 1e-5)
    bad, _ = R.layernorm(x, torch.ones(256, dtype=F64), torch.zeros(256, dtype=F64), 1e-5, eps_scale=10)
    assert ((bad - ok).abs() / e).max() > 1
    q, k, v = (torch.randn(2, 9, 256, generator=g, dtype=F64) for _ in range(3))
    ok, e = R.mha(q, k, v, None, 0.125)
    bad, _ = R.mha(q, k, v, None, 0.125, drop_last_key=True)
    assert ((bad - ok).abs() / e).max() > 1
    assert np.isclose(R.gamma(1), R.U / (1 - R.U))
