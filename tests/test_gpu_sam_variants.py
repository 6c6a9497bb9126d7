"""GPU: SAM ViT-L and ViT-B (head dim 64) in the ISM segmentor.  The head-dim-64 instantiations of the three SAM attention
kernels against the reference formula (image_encoder.py:224-240, 325-361), the full ViT-B / ViT-L encoders against the vendored
reference module's CPU output (tests/golden/sam_vit{b,l}.pt, tools/make_golden.py), batch independence, and the ISM CLI with
--sam_model_type vit_b chained into the PEM CLI."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import sam_oracle as so      # noqa: E402


def _ref_attention(q, k, v, rel_h, rel_w, S, scale):
    """q, k, v (n, S*S, D) -> (n, S*S, D): softmax(q*scale k^T + q.Rh + q.Rw) v in the device's fp32"""
    n, L, D = q.shape
    attn = (q * scale) @ k.transpose(-2, -1)
    Rh, Rw = so.rel_pos_table(S, rel_h).to(q.device), so.rel_pos_table(S, rel_w).to(q.device)
    rq = q.reshape(n, S, S, D)
    attn = (attn.view(-1, S, S, S, S) + torch.einsum("bhwc,hkc->bhwk", rq, Rh)[:, :, :, :, None] +
            torch.einsum("bhwc,wkc->bhwk", rq, Rw)[:, :, :, None, :]).view(-1, L, L).softmax(dim=-1)
    return attn @ v


def _split_heads(qkv, nW, L, H, D):
    return qkv.view(nW, L, 3, H, D).permute(2, 0, 3, 1, 4).reshape(3, nW * H, L, D).unbind(0)


def _global_case(B, H, D, seed):
    S = 64
    L = S * S
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(B * L, 3 * H * D, generator=g) * 1.5).bfloat16()
    rel_h = torch.randn(2 * S - 1, D, generator=g) * 0.2
    rel_w = torch.randn(2 * S - 1, D, generator=g) * 0.2
    return qkv, rel_h, rel_w


@pytest.mark.parametrize("H", [12, 16])
def test_attn_global_tc_head_dim_64(H):
    """the D = 64 global attention against the fp32 formula on the same bf16-rounded q, k, v, at the tolerances of the D = 80
    test (test_gpu_kernels.py::test_attn_global_tensor_core)"""
    from sam6d_b200 import ops
    B, S, D = 2, 64, 64
    L = S * S
    qkv, rel_h, rel_w = _global_case(B, H, D, 64 + H)
    q, k, v = _split_heads(qkv.float().cuda(), B, L, H, D)
    ref = _ref_attention(q, k, v, rel_h, rel_w, S, D ** -0.5).view(B, H, L, D).permute(0, 2, 1, 3).reshape(B * L, H * D).cpu()
    del q, k, v
    qd = qkv.cuda()
    vt = ops.transpose_tokens(qd, 2 * H * D, H * D, B, L)
    blob = ops.pack_rel_pos(rel_h.cuda(), rel_w.cuda(), slab_rows=128)
    assert blob.numel() == 2 * 128 * 64                                     # one slab per table at D = 64
    for odt in (torch.float32, torch.bfloat16):
        got = ops.attn_global_tc(qd, vt, blob, B, H, S, D ** -0.5, out_dtype=odt, D=D).cpu().float()
        err = (got - ref).abs()
        print(f"attn_global_tc D=64 H={H} {odt}: max err {err.max().item():.3e}, mean err {err.mean().item():.3e}")
        torch.testing.assert_close(got, ref, atol=6e-2, rtol=2e-2)
        assert err.mean().item() < 3e-3


def test_attn_global_tc_ex_head_dim_80_is_the_old_entry_point():
    """sam6d_attn_global_tc and sam6d_attn_global_tc_ex(head_dim=80) are the same launch: bit-identical outputs"""
    from sam6d_b200 import _lib, ops
    B, H, D, S = 2, 4, 80, 64
    L = S * S
    qkv, rel_h, rel_w = _global_case(B, H, D, 80)
    qd = qkv.cuda()
    vt = ops.transpose_tokens(qd, 2 * H * D, H * D, B, L)
    blob = ops.pack_rel_pos(rel_h.cuda(), rel_w.cuda(), slab_rows=128)
    for odt in (torch.float32, torch.bfloat16):
        a = torch.full((B * L, H * D), float("nan"), dtype=odt, device="cuda")
        b = torch.full_like(a, float("nan"))
        bf = int(odt == torch.bfloat16)
        _lib.call("sam6d_attn_global_tc", qd, qd.shape[1], vt, vt.shape[1], blob, B, H, S, D ** -0.5, a, bf, H * D)
        _lib.call("sam6d_attn_global_tc_ex", qd, qd.shape[1], vt, vt.shape[1], blob, B, H, S, 80, D ** -0.5, b, bf, H * D)
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)
        torch.testing.assert_close(ops.attn_global_tc(qd, vt, blob, B, H, S, D ** -0.5, out_dtype=odt), a, atol=0, rtol=0)


def test_attn_global_tc_ex_rejects_other_head_dims():
    from sam6d_b200 import _lib, ops
    B, H, S = 1, 2, 64
    qkv = torch.zeros(B * S * S, 3 * H * 96, dtype=torch.bfloat16, device="cuda")
    vt = ops.transpose_tokens(qkv, 2 * H * 96, H * 96, B, S * S)
    blob = torch.zeros(4 * 128 * 64, dtype=torch.bfloat16, device="cuda")
    for D in (32, 96, 128):
        with pytest.raises(_lib.Sam6dError, match="invalid argument"):
            ops.attn_global_tc(qkv, vt, blob, B, H, S, 0.1, D=D)


def test_attn_tc_sam_window_head_dim_64():
    """windowed tensor-core attention with the decomposed rel-pos bias (14 x 14 windows) at D = 64, at the tolerances of the
    D = 80 windowed test (test_gpu_kernels.py::test_attn_tc_sam_window)"""
    from sam6d_b200 import ops
    nW, S, H, D = 4, 14, 3, 64
    L = S * S
    g = torch.Generator().manual_seed(164)
    qkv = torch.randn(nW * L, 3 * H * D, generator=g)
    rel_h = torch.randn(2 * S - 1, D, generator=g) * 0.1
    rel_w = torch.randn(2 * S - 1, D, generator=g) * 0.1
    qkv_b = qkv.bfloat16()
    q, k, v = _split_heads(qkv_b.float(), nW, L, H, D)
    ref = _ref_attention(q, k, v, rel_h, rel_w, S, D ** -0.5).view(nW, H, L, D).permute(0, 2, 1, 3).reshape(nW * L, H * D)
    N1 = (L + 15) // 16 * 16
    vt = torch.zeros(nW * H * D, N1, dtype=torch.bfloat16)
    vt[:, :L] = qkv_b[:, 2 * H * D:].view(nW, L, H, D).permute(0, 2, 3, 1).reshape(nW * H * D, L)
    qk = qkv_b[:, :2 * H * D].contiguous()
    blob = ops.pack_rel_pos(rel_h.cuda(), rel_w.cuda())
    assert blob.numel() == 2 * 32 * 64                                      # one slab per table at D = 64
    for odt in (torch.float32, torch.bfloat16):
        got = ops.attn_tc(qk.cuda(), 0, qk.cuda(), H * D, vt.cuda(), nW, H, L, L, D, D ** -0.5, rel=(blob, S, S), out_dtype=odt).cpu().float()
        torch.testing.assert_close(got, ref, atol=2e-2, rtol=2e-2)
        assert (got - ref).abs().mean().item() < 3e-3


@pytest.mark.parametrize("nW,S,nH", [(3, 14, 4), (1, 64, 2), (2, 9, 1)])
def test_attn_relpos_kernel_head_dim_64(nW, S, nH):
    """the fp32 comparator at D = 64 on the shapes of test_gpu_sam.py::test_attn_relpos_kernel"""
    from sam6d_b200 import ops
    D = 64
    g = torch.Generator().manual_seed(100 + S)
    qkv = torch.randn(nW * S * S, 3 * nH * D, generator=g)
    rel_h = torch.randn(2 * S - 1, D, generator=g) * 0.1
    rel_w = torch.randn(2 * S - 1, D, generator=g) * 0.1
    q, k, v = _split_heads(qkv, nW, S * S, nH, D)
    ref = _ref_attention(q, k, v, rel_h, rel_w, S, D ** -0.5).view(nW, nH, S * S, D).permute(0, 2, 1, 3).reshape(nW * S * S, nH * D)
    got = ops.attn_relpos(qkv.cuda(), nW, S, S, nH, rel_h.cuda(), rel_w.cuda(), D ** -0.5).cpu()
    torch.testing.assert_close(got, ref, atol=2e-5, rtol=1e-4)
    got_bf = ops.attn_relpos(qkv.cuda(), nW, S, S, nH, rel_h.cuda(), rel_w.cuda(), D ** -0.5, out_dtype=torch.bfloat16).cpu()
    torch.testing.assert_close(got_bf.float(), got.bfloat16().float(), atol=0, rtol=0)


def _encoder(name, precision):
    from sam6d_b200.sam import build_image_encoder
    return build_image_encoder(name, precision=precision).cuda().eval()


# (rms error / output std, cosine) bounds: the drift measured on an H100 80GB HBM3 plus margin -- fp32 1.5e-6 / 1.6e-6 and
# cosine 1 - 1e-7 (vit_b / vit_l), bf16 6.0e-3 / 6.4e-3 and cosine 0.99998 -- tighter than the ViT-H test's 2e-3 / 0.99999 (fp32)
# and 0.12 / 0.993 (bf16)
BOUNDS = {"fp32": (2e-5, 0.999999), "bf16": (2e-2, 0.9999)}


@pytest.mark.parametrize("name,golden", [("vit_b", "sam_vitb.pt"), ("vit_l", "sam_vitl.pt")])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_encoder_matches_reference_golden(golden_dir, name, golden, precision):
    """the full ViT-B (12 blocks) / ViT-L (24 blocks) of build_sam.py:27-44 on one 1024 x 1024 frame against the vendored
    reference module's CPU output, with the metric of test_gpu_sam.py::test_vit_h_32_blocks_matches_reference_golden"""
    from sam6d_b200.sam import VIT_CONFIGS
    gold = torch.load(os.path.join(golden_dir, golden), weights_only=False)
    cfg = gold["meta"]["cfg"]
    assert cfg == VIT_CONFIGS[name]
    enc = _encoder(name, precision)
    enc.load_state_dict(so.make_state_dict(seed=gold["meta"]["seed"], **cfg), strict=True)
    img = so.make_images(B=1, seed=gold["meta"]["img_seed"])
    out = enc(img.cuda()).cpu()
    assert out.shape == (1, 256, 64, 64)
    ref = gold["out_sub"]
    err = (out[:, :, ::4, ::4] - ref).abs()
    rel_rms = (err.pow(2).mean().sqrt() / gold["out_std"]).item()
    cos = torch.nn.functional.cosine_similarity(out[:, :, ::4, ::4].flatten(), ref.flatten(), dim=0).item()
    print(f"SAM {name} {cfg['depth']} blocks {precision}: max err {err.max().item():.3e}, rms err / output std {rel_rms:.3e}, "
          f"cosine {cos:.7f}, |ref| max {gold['out_abs_max']:.2f} std {gold['out_std']:.3f}")
    assert torch.isfinite(out).all()
    rms_bound, cos_bound = BOUNDS[precision]
    assert rel_rms < rms_bound and cos > cos_bound


def test_vit_b_batch_and_independence():
    """two frames in one batch give the same ViT-B embeddings as one at a time (no cross-image leakage through the window maps
    or the head-dim-64 global attention)"""
    from sam6d_b200.sam import VIT_CONFIGS
    enc = _encoder("vit_b", "bf16")
    enc.load_state_dict(so.make_state_dict(seed=2, **VIT_CONFIGS["vit_b"]), strict=True)
    img = so.make_images(B=2, seed=5).cuda()
    both = enc(img)
    one = enc(img[1:2].contiguous())
    torch.testing.assert_close(both[1:2], one, atol=1e-5, rtol=1e-5)
    assert torch.isfinite(both).all()


def _write_ply(path, verts_mm, faces, colors):
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\n"
                 "end_header\n" % (len(verts_mm), len(faces)))
        for v, c in zip(verts_mm, colors):
            fh.write("%f %f %f %d %d %d\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
        for f in faces:
            fh.write("3 %d %d %d\n" % tuple(f))


def test_ism_cli_vit_b_then_pem_cli(tmp_path, golden_dir):
    """the ISM CLI on the ViT-B backbone (--sam_model_type vit_b, seeded weights) chained into the PEM CLI, as
    test_gpu_cli.py::test_ism_cli_then_pem_cli does for the default ViT-H"""
    import cv2
    from scipy.spatial import ConvexHull
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, pem_run_inference_custom as pem_cli, render_point_templates as rpt
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
    assert ism_cli.main(common + ["--sam_model_type", "vit_b", "--random_weights", "--stability_score_thresh", "0.0",
                                  "--pred_iou_thresh", "-10", "--confidence_thresh", "-1", "--points_per_side", "8"]) == 0
    dets = json.load(open(os.path.join(out, "sam6d_results", "detection_ism.json")))
    print(f"ISM CLI (vit_b): {len(dets)} detections")
    assert len(dets) >= 1
    for d in dets:
        assert set(["scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation"]) <= set(d)
        assert d["segmentation"]["size"] == [480, 640] and sum(d["segmentation"]["counts"]) == 480 * 640
        assert len(d["bbox"]) == 4 and np.isfinite(d["score"])
    np.random.seed(0)
    assert pem_cli.main(common + ["--seg_path", os.path.join(out, "sam6d_results", "detection_ism.json"), "--random_weights",
                                  "--det_score_thresh", "-1"]) == 0
    res = json.load(open(os.path.join(out, "sam6d_results", "detection_pem.json")))
    assert len(res) <= len(dets)
    for r in res:
        R = np.array(r["R"])
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-4) and np.isfinite(np.array(r["t"])).all()
