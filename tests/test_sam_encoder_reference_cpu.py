"""CPU: the float64 restatements that tests/test_gpu_sam_encoder_kernels.py holds the encoder's kernels to
(tests/_sam_encoder_ref.py) against oracle/sam_oracle.py, which is pinned to the reference module; and the encoder's static
gather maps (ImageEncoderViT._index_maps) against the reference's window_partition / window_unpartition and the 3 x 3 neck
convolution, exactly.  A wrong restatement would make every bound of the GPU file meaningless."""
import types

import pytest
import torch
import torch.nn.functional as F

import _sam_encoder_ref as er   # noqa: E402
from oracle import sam_oracle as so
from sam6d_b200.sam import ImageEncoderViT

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("Hs,Ws,H,D", [(14, 14, 2, 80), (9, 20, 3, 64), (12, 16, 2, 64), (5, 5, 4, 80)])
def test_relpos_attention_matches_oracle(Hs, Ws, H, D):
    """relpos_attention (explicit index tables) == sam_oracle.attention (get_rel_pos / einsum form) with an identity proj"""
    g = _g(Hs * 100 + Ws)
    C, nW = H * D, 3
    x = torch.randn(nW, Hs, Ws, C, generator=g, dtype=F64)
    sd = {"a.qkv.weight": torch.randn(3 * C, C, generator=g, dtype=F64) / C ** 0.5,
          "a.qkv.bias": torch.randn(3 * C, generator=g, dtype=F64) * 0.1,
          "a.proj.weight": torch.eye(C, dtype=F64), "a.proj.bias": torch.zeros(C, dtype=F64),
          "a.rel_pos_h": torch.randn(2 * Hs - 1, D, generator=g, dtype=F64) * 0.5,
          "a.rel_pos_w": torch.randn(2 * Ws - 1, D, generator=g, dtype=F64) * 0.5}
    ref = so.attention(sd, "a", x, H)
    qkv = F.linear(x.reshape(nW, Hs * Ws, C), sd["a.qkv.weight"], sd["a.qkv.bias"]).view(nW, Hs * Ws, 3, H, D)
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    got = er.relpos_attention(q, k, v, sd["a.rel_pos_h"], sd["a.rel_pos_w"], Hs, Ws, D ** -0.5)
    got = got.permute(0, 2, 1, 3).reshape(nW, Hs, Ws, C)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    # the bias really is asymmetric in (h, w) here: swapping the tables changes the answer
    if Hs == Ws:
        wrong = torch.softmax((q * D ** -0.5) @ k.transpose(-1, -2) +
                              er.decomposed_bias(q, sd["a.rel_pos_w"], sd["a.rel_pos_h"], Hs, Ws), -1) @ v
        assert (wrong.permute(0, 2, 1, 3).reshape(nW, Hs, Ws, C) - ref).abs().max() > 1e-3


def test_layer_norm_matches_oracle():
    """er.layer_norm == F.layer_norm (Block.norm1 / norm2) and == sam_oracle.layernorm2d (the neck's LayerNorm2d, channel-last)"""
    g = _g(5)
    x = torch.randn(7, 256, generator=g, dtype=F64) * 3 + 50
    w, b = torch.randn(256, generator=g, dtype=F64), torch.randn(256, generator=g, dtype=F64)
    got = er.layer_norm(x, w, b, 1e-6)
    torch.testing.assert_close(got, F.layer_norm(x, (256,), w, b, 1e-6), rtol=1e-12, atol=1e-12)
    img = x.t().reshape(1, 256, 7, 1)
    torch.testing.assert_close(got, so.layernorm2d(img, w, b, 1e-6).reshape(256, 7).t(), rtol=1e-12, atol=1e-12)


def _maps(B, G=64, ws=14):
    return ImageEncoderViT._index_maps(types.SimpleNamespace(_maps={}), B, G, ws, "cpu")


@pytest.mark.parametrize("B", [1, 2])
def test_partition_maps_match_reference(B):
    """part / unpart of the encoder == window_partition (F.pad 64 -> 70) / window_unpartition on token ids, exactly"""
    m = _maps(B)
    part, (Hp, Wp) = er.partition_ids(B, 64, 14)
    assert (Hp, Wp) == (70, 70) and m["nwin"] == 5
    assert part.shape == (B, 25 * 196)
    assert torch.equal(m["part"].long(), part)
    assert int((part[0] < 0).sum()) == 70 * 70 - 64 * 64
    assert torch.equal(m["unpart"].long(), er.unpartition_ids(B, 64, 14))
    # unpartition undoes partition: every grid token comes back from the window slot it was sent to
    tok = torch.arange(64 * 64)
    assert torch.equal(part[0][m["unpart"][0].long()], tok)


def test_neck_taps_match_conv_neighbourhoods():
    """the 9 shifted gathers of the neck's 3 x 3 conv == the neighbourhoods F.conv2d(padding=1) multiplies by weight[:, :, kh, kw]"""
    m = _maps(2)
    ref = er.conv3x3_taps(64)
    assert len(m["taps"]) == 9
    for t in range(9):
        assert torch.equal(m["taps"][t][0].long(), ref[t]), f"tap {t}"
        assert torch.equal(m["taps"][t][1], m["taps"][t][0])
    # a 3 x 3 conv evaluated through the taps == F.conv2d(padding=1)
    g = _g(9)
    x = torch.randn(1, 5, 64, 64, generator=g, dtype=F64)
    w = torch.randn(4, 5, 3, 3, generator=g, dtype=F64)
    rows = x[0].reshape(5, -1).t()
    acc = torch.zeros(64 * 64, 4, dtype=F64)
    for t in range(9):
        idx = m["taps"][t][0].long()
        shifted = torch.where((idx >= 0)[:, None], rows[idx.clamp_min(0)], torch.zeros_like(rows))
        acc += shifted @ w[:, :, t // 3, t % 3].t()
    torch.testing.assert_close(acc.t().reshape(1, 4, 64, 64), F.conv2d(x, w, padding=1), rtol=1e-12, atol=1e-12)
