"""GPU: the ISM descriptor branch (SURVEY.md 8f row N2: sam6d_b200/dinov2.py, csrc/ism_desc.cu, the 257-token attention) against
tests/golden/dinov2.pt -- outputs of the reference's OWN vit_large (dinov2_vitl14 architecture), CropResizePad, CustomDINOv2 and
MaskedPatch_MatrixSimilarity on seeded weights and a synthetic 6-proposal frame (tools/make_golden_dinov2.py)."""
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import dinov2_oracle as do, ism_oracle as io      # noqa: E402


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "dinov2.pt"), weights_only=False)


@pytest.fixture(scope="module")
def desc(gold):
    from sam6d_b200.dinov2 import CustomDINOv2
    d = CustomDINOv2().cuda().eval()
    d.model.load_state_dict(do.make_state_dict(seed=gold["meta"]["seed"]), strict=True)
    return d


def test_crop_resize_pad_bit_exact(gold, desc):
    image, masks, boxes = do.make_proposals(P=gold["meta"]["P"], seed=gold["meta"]["seed"])
    rgbs = desc.process_rgb_proposals(image.numpy(), masks.cuda(), boxes.cuda()).cpu()
    pm = desc.process_masks_proposals(masks.cuda(), boxes.cuda()).cpu()
    assert torch.equal((pm > 0.5).to(torch.uint8), gold["pmasks_packed"])
    torch.testing.assert_close(rgbs[:, :, ::7, ::7], gold["rgbs_sub"], atol=1e-6, rtol=0)
    torch.testing.assert_close(rgbs.double().sum(dim=(1, 2, 3)), gold["rgbs_sum"], atol=1e-2, rtol=1e-6)
    # against the oracle on boxes the fixture does not hold: tiny, exactly square, one-pixel-short squares, full frame
    g = torch.Generator().manual_seed(3)
    extra = torch.tensor([[10, 10, 13, 12], [100, 50, 200, 150], [0, 0, 639, 479], [5, 5, 118, 118], [300, 200, 523, 423], [7, 300, 8, 470]])
    m2 = (torch.rand(len(extra), 480, 640, generator=g) > 0.3).float()
    want = do.process_rgb_proposals(image, m2.clone(), extra)
    got = desc.process_rgb_proposals(image.numpy(), m2.cuda(), extra.cuda()).cpu()
    torch.testing.assert_close(got, want, atol=1e-6, rtol=0)
    assert torch.equal(desc.process_masks_proposals(m2.cuda(), extra.cuda()).cpu(), do.process_masks_proposals(m2.clone(), extra))


def test_vit_l14_descriptors_match_reference(gold, desc):
    """cls tokens and masked, normalised patch tokens of the 24-block ViT-L/14 (257-token attention = 256 keys on wgmma + the
    class token merged by log-sum-exp); bf16 operands, so the bound is the measured drift plus margin, stated relative to the
    descriptor scale; the patch-validity pattern is exact"""
    image, masks, boxes = do.make_proposals(P=gold["meta"]["P"], seed=gold["meta"]["seed"])
    cls, pf = desc(image.numpy(), SimpleNamespace(masks=masks.cuda(), boxes=boxes.cuda()))
    cls, pf = cls.cpu(), pf.cpu()
    assert cls.shape == (6, 1024) and pf.shape == (6, 256, 1024)
    cos = torch.nn.functional.cosine_similarity(cls, gold["cls"], dim=1)
    rel = (cls - gold["cls"]).norm(dim=1) / gold["cls"].norm(dim=1)
    print(f"DINOv2 ViT-L/14 cls tokens: cosine min {cos.min().item():.6f}, relative L2 error max {rel.max().item():.3e}")
    assert cos.min().item() > 0.999 and rel.max().item() < 4e-2
    assert torch.equal(desc.last_valid.cpu().bool(), gold["keep"])
    sub = pf[:, ::5, :]
    err = (sub - gold["patch_sub"]).abs()
    print(f"masked patch tokens: max err {err.max().item():.3e} (unit-norm rows), zero rows exact: {bool((sub[~gold['keep'][:, ::5]] == 0).all())}")
    assert err.max().item() < 1e-2 and (sub[~gold["keep"][:, ::5]] == 0).all()


def test_appearance_score_and_visible_ratio(gold, desc):
    from sam6d_b200.dinov2 import MaskedPatch_MatrixSimilarity
    g = torch.Generator().manual_seed(2)
    P, N, C = 9, 256, 1024
    q = torch.nn.functional.normalize(torch.randn(P, N, C, generator=g), dim=-1)
    r = torch.nn.functional.normalize(q.roll(3, dims=1) + 0.8 * torch.randn(P, N, C, generator=g), dim=-1)
    q[:, 200:, :] = 0                       # masked query patches
    r[:, :40, :] = 0                        # masked template patches
    q[8] = 0                                # a proposal without any valid patch
    m = MaskedPatch_MatrixSimilarity()
    appe, vis = m.scores(q.cuda(), r.cuda(), 0.5)
    qb, rb = q.bfloat16().float(), r.bfloat16().float()
    torch.testing.assert_close(appe.cpu(), io.appearance_score(qb, rb), atol=2e-4, rtol=0)
    torch.testing.assert_close(vis.cpu(), io.visible_ratio(qb, rb, 0.5), atol=1e-6, rtol=0)
    # and against the reference numbers of the fixture (fp32 descriptors -> bf16 operands: looser)
    image, masks, boxes = do.make_proposals(P=gold["meta"]["P"], seed=gold["meta"]["seed"])
    _, pf = desc(image.numpy(), SimpleNamespace(masks=masks.cuda(), boxes=boxes.cuda()))
    appe, vis = m.scores(pf, pf.roll(1, dims=0), 0.5)
    print("appearance", appe.cpu().tolist(), gold["appe"].tolist(), "visible", vis.cpu().tolist(), gold["vis"].tolist())
    torch.testing.assert_close(appe.cpu(), gold["appe"], atol=2e-2, rtol=0)
    torch.testing.assert_close(vis.cpu(), gold["vis"], atol=0.1, rtol=0)


def test_attention_257_tokens_against_softmax(desc):
    """the 256-key tensor-core pass + class-token merge equals a plain softmax over 257 keys"""
    from sam6d_b200 import ops
    B, H, S, d = 3, 16, 257, 64
    C = H * d
    g = torch.Generator().manual_seed(0)
    qkv = (torch.randn(B * S, 3 * C, generator=g) * 0.7).bfloat16()
    q, k, v = qkv[:, :C].float().view(B, S, H, d), qkv[:, C:2 * C].float().view(B, S, H, d), qkv[:, 2 * C:].float().view(B, S, H, d)
    att = torch.softmax(torch.einsum("bnhd,bmhd->bhnm", q, k) * d ** -0.5, dim=-1)
    ref = torch.einsum("bhnm,bmhd->bnhd", att, v).reshape(B * S, C)
    qk = qkv[:, :2 * C].contiguous().cuda()
    vt = ops.transpose_tokens(qkv.cuda(), 2 * C, C, B, S)                       # (B*C, 272) = V^T per image
    got = desc.model._attention(qk, vt, B, S, C).float().cpu()
    torch.testing.assert_close(got, ref, atol=2e-2, rtol=2e-2)
