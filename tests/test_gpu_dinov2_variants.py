"""GPU: the DINOv2 ViT-S/14, ViT-B/14 and ViT-g/14 descriptor backbones (sam6d_b200/dinov2.py) and the SwiGLU epilogue of
sam6d_gemm_tma (act=3) that ViT-g's FFN runs on.  Descriptors are checked against tests/golden/dinov2_variants.pt -- outputs of the
reference's own vit_small / vit_base / vit_giant2(ffn_layer="swiglufused") on seeded weights and the synthetic 6-proposal frame
(tools/make_golden_dinov2_variants.py) -- and the scoring kernels at the three new descriptor widths against oracle/ism_oracle.py."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import dinov2_oracle as do, dinov2_variants_oracle as dvo, ism_oracle as io      # noqa: E402

# cls tokens: min cosine / max relative L2 error; patch tokens (unit rows): max abs error.  Bounds are the drift measured with bf16
# operands, fp32 accumulation and residual stream, plus margin (ViT-L/14's are in tests/test_gpu_dinov2.py).  Measured on an
# H100 80GB HBM3 at 700 W: ViT-S cosine 0.999978 / rel 6.7e-3 / patch 1.1e-3, ViT-B 0.999978 / 6.7e-3 / 1.1e-3, ViT-g (40
# blocks) 0.999913 / 1.3e-2 / 1.4e-3.
BOUNDS = {
    "dinov2_vits14": (0.9999, 2e-2, 4e-3),
    "dinov2_vitb14": (0.9999, 2e-2, 4e-3),
    "dinov2_vitg14": (0.9996, 4e-2, 5e-3),
}


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "dinov2_variants.pt"), weights_only=False)


def _swiglu_ref(x, w12, b12):
    """SwiGLUFFN's hidden activation (ISM/model/layers/swiglu_ffn.py:29-32) in fp32 on the operands the kernel reads"""
    x1, x2 = (x.float() @ w12.bfloat16().float().t() + b12).chunk(2, dim=-1)
    return F.silu(x1) * x2


@pytest.mark.parametrize("M,K,H", [(6 * 257, 1536, 4096), (257, 1536, 4096), (1, 384, 256), (130, 768, 512), (2049, 64, 128)])
def test_swiglu_gemm_against_torch(M, K, H):
    """gemm_tma(act=3) on the interleaved w12 equals silu(x w1^T + b1) * (x w2^T + b2) computed in fp32 by torch on the same
    bf16-rounded operands, within one bf16 ulp (the kernel rounds its result to bf16 once); ragged M, K of one k-block"""
    from sam6d_b200 import ops
    g = torch.Generator().manual_seed(M + K + H)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w12 = (torch.randn(2 * H, K, generator=g) / K ** 0.5).cuda()
    b12 = (0.5 * torch.randn(2 * H, generator=g)).cuda()
    got = ops.gemm_tma(x, ops.pack_swiglu_rows(w12).bfloat16(), ops.pack_swiglu_rows(b12), act=ops.ACT_SWIGLU)
    assert got.shape == (M, H) and got.dtype == torch.bfloat16
    want = _swiglu_ref(x, w12, b12)
    err = (got.float() - want).abs()
    bound = 2 ** -7 * want.abs() + 1e-4            # one bf16 ulp of the result plus fp32 summation-order noise (measured: <= half)
    print(f"SwiGLU GEMM M={M} K={K} H={H}: max err {err.max().item():.3e}, max err / bound {(err / bound).max().item():.3f}")
    assert (err <= bound).all()
    # the interleave matters: the reference's [gate; up] order fed unpacked mixes gate and up units of different hidden indices
    if H > 128:
        wrong = ops.gemm_tma(x, w12.bfloat16(), b12, act=ops.ACT_SWIGLU).float()
        assert (wrong - want).abs().max().item() > 10 * err.max().item() + 1e-2


def test_swiglu_gemm_argument_checks():
    from sam6d_b200 import _lib, ops
    x = torch.randn(64, 128, device="cuda").bfloat16()
    w = torch.randn(512, 128, device="cuda").bfloat16()
    b = torch.zeros(512, device="cuda")
    with pytest.raises(_lib.Sam6dError):                    # N % 256 != 0
        ops.gemm_tma(x, w[:384], b[:384], act=ops.ACT_SWIGLU)
    with pytest.raises(_lib.Sam6dError):                    # bias required
        ops.gemm_tma(x, w, None, act=ops.ACT_SWIGLU)
    with pytest.raises(_lib.Sam6dError):                    # fp32 output
        ops.gemm_tma(x, w, b, act=ops.ACT_SWIGLU, out=torch.empty(64, 256, device="cuda"))
    with pytest.raises(_lib.Sam6dError):                    # residual
        ops.gemm_tma(x, w, b, act=ops.ACT_SWIGLU, residual=torch.zeros(64, 256, device="cuda").bfloat16())


def _descriptor(name, seed):
    from sam6d_b200.dinov2 import CustomDINOv2
    with torch.device("cuda"):                              # ViT-g has 1.1 G parameters: initialise them on the device
        d = CustomDINOv2(name).eval()
    d.model.load_state_dict(dvo.make_state_dict(name, seed=seed), strict=True)
    return d


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vitb14", "dinov2_vitg14"])
def test_descriptors_match_reference(gold, name):
    """cls tokens and masked, normalised patch tokens of the full-depth backbone against the reference's module; bf16 operands,
    so the bounds are the measured drift plus margin; the patch-validity pattern is exact"""
    g, meta = gold["models"][name], gold["meta"]
    d = _descriptor(name, meta["seed"])
    image, masks, boxes = do.make_proposals(P=meta["P"], seed=meta["seed"])
    cls, pf = d(image.numpy(), SimpleNamespace(masks=masks.cuda(), boxes=boxes.cuda()))
    cls, pf = cls.cpu(), pf.cpu()
    C = g["arch"]["embed_dim"]
    assert cls.shape == (6, C) and pf.shape == (6, 256, C)
    cos = F.cosine_similarity(cls, g["cls"], dim=1)
    rel = (cls - g["cls"]).norm(dim=1) / g["cls"].norm(dim=1)
    sub = pf[:, ::meta["patch_step"], ::meta["channel_step"]]
    err = (sub - g["patch_sub"]).abs()
    print(f"DINOv2 {name} cls tokens: cosine min {cos.min().item():.6f}, relative L2 error max {rel.max().item():.3e}; "
          f"masked patch tokens: max err {err.max().item():.3e}")
    cos_min, rel_max, patch_max = BOUNDS[name]
    assert torch.equal(d.last_valid.cpu().bool(), g["keep"])
    # every token, not only the fixture's subsample: masked rows exactly zero, the others unit-norm
    assert (pf[~g["keep"]] == 0).all() and ((pf[g["keep"]].norm(dim=-1) - 1).abs() < 1e-4).all()
    assert cos.min().item() > cos_min and rel.max().item() < rel_max
    assert err.max().item() < patch_max
    from sam6d_b200.dinov2 import MaskedPatch_MatrixSimilarity
    appe, vis = MaskedPatch_MatrixSimilarity().scores(pf.cuda(), pf.roll(1, dims=0).cuda(), 0.5)
    print("appearance", appe.cpu().tolist(), g["appe"].tolist(), "visible", vis.cpu().tolist(), g["vis"].tolist())
    torch.testing.assert_close(appe.cpu(), g["appe"], atol=2e-2, rtol=0)
    torch.testing.assert_close(vis.cpu(), g["vis"], atol=0.1, rtol=0)


@pytest.mark.parametrize("C", [384, 768, 1536])
def test_template_score_at_descriptor_width(C):
    from sam6d_b200 import ism
    q, r = io.make_descriptors(P=200, O=21, T=42, C=C, seed=C)
    idx_sel, pred_obj, sem, best_t, scores, _ = io.compute_semantic_score(q, r)
    sim = ism.PairwiseSimilarity()(q.cuda(), r.cuda()).cpu()
    torch.testing.assert_close(sim, scores, atol=2e-6, rtol=1e-5)
    g_sel, g_obj, g_sem, g_t = ism.compute_semantic_score(q.cuda(), r.cuda())
    assert torch.equal(g_sel.cpu(), idx_sel) and torch.equal(g_obj.cpu(), pred_obj) and torch.equal(g_t.cpu(), best_t)
    torch.testing.assert_close(g_sem.cpu(), sem, atol=2e-6, rtol=1e-5)


@pytest.mark.parametrize("C", [384, 768, 1536])
def test_appearance_score_at_descriptor_width(C):
    """MaskedPatch_MatrixSimilarity.scores (batched 256 x 256 x C GEMM + reduction) against the reference formulas on the same
    bf16-rounded descriptors, with masked query / template patches and a proposal without any valid patch"""
    from sam6d_b200.dinov2 import MaskedPatch_MatrixSimilarity
    g = torch.Generator().manual_seed(C)
    P, N = 9, 256
    q = F.normalize(torch.randn(P, N, C, generator=g), dim=-1)
    r = F.normalize(q.roll(3, dims=1) + 0.8 * torch.randn(P, N, C, generator=g), dim=-1)
    q[:, 200:, :] = 0
    r[:, :40, :] = 0
    q[8] = 0
    appe, vis = MaskedPatch_MatrixSimilarity().scores(q.cuda(), r.cuda(), 0.5)
    qb, rb = q.bfloat16().float(), r.bfloat16().float()
    torch.testing.assert_close(appe.cpu(), io.appearance_score(qb, rb), atol=2e-4, rtol=0)
    torch.testing.assert_close(vis.cpu(), io.visible_ratio(qb, rb, 0.5), atol=1e-6, rtol=0)


def _write_ply(path, verts_mm, faces, colors):
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                 % (len(verts_mm), len(faces)))
        for v, c in zip(verts_mm, colors):
            fh.write("%f %f %f %d %d %d\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
        for f in faces:
            fh.write("3 %d %d %d\n" % tuple(f))


def test_ism_cli_dinov2_vits14(tmp_path, golden_dir):
    """the ISM CLI with --dinov2_model dinov2_vits14 (seeded weights) on the example frame and point-splat templates"""
    import cv2
    from scipy.spatial import ConvexHull
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, render_point_templates as rpt
    gold = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    out = str(tmp_path)
    cv2.imwrite(os.path.join(out, "rgb.png"), gold["rgb"].numpy()[:, :, ::-1])
    cv2.imwrite(os.path.join(out, "depth.png"), gold["depth"].numpy().astype(np.uint16))
    json.dump(dict(cam_K=gold["cam_K"], depth_scale=gold["depth_scale"]), open(os.path.join(out, "camera.json"), "w"))
    pts_mm = gold["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts_mm)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    cad = os.path.join(out, "obj.ply")
    _write_ply(cad, pts_mm[hull.vertices], np.array([[remap[a] for a in s] for s in hull.simplices]),
               np.random.RandomState(0).randint(40, 255, (len(hull.vertices), 3)))
    rpt.main(["--cad_path", cad, "--output_dir", out, "--size", "192"])
    common = ["--output_dir", out, "--cad_path", cad, "--rgb_path", os.path.join(out, "rgb.png"), "--depth_path", os.path.join(out, "depth.png"),
              "--cam_path", os.path.join(out, "camera.json")]
    assert ism_cli.main(common + ["--dinov2_model", "dinov2_vits14", "--random_weights", "--stability_score_thresh", "0.0",
                                  "--pred_iou_thresh", "-10", "--confidence_thresh", "-1", "--points_per_side", "8"]) == 0
    dets = json.load(open(os.path.join(out, "sam6d_results", "detection_ism.json")))
    print(f"ISM CLI (dinov2_vits14): {len(dets)} detections")
    assert len(dets) >= 1
    for d in dets:
        assert set(["scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation"]) <= set(d)
        assert d["segmentation"]["size"] == [480, 640] and sum(d["segmentation"]["counts"]) == 480 * 640
        assert len(d["bbox"]) == 4 and np.isfinite(d["score"]) and 0.0 <= d["score"] <= 1.0
