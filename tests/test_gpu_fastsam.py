"""GPU: the FastSAM segmentor (sam6d_b200/fast_sam.py, csrc/conv_tc.cu, csrc/yolo.cu) against the fp32 CPU restatement
oracle/fastsam_oracle.py, on seeded weights (synth.make_fastsam_state_dict) and synthetic frames."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U_FP32 = 2.0 ** -24          # unit roundoff of fp32
U_BF16 = 2.0 ** -8           # unit roundoff of bf16 (8 significand bits)


@pytest.fixture(scope="module")
def sd():
    from sam6d_b200 import synth
    return synth.make_fastsam_state_dict(1)


@pytest.fixture(scope="module")
def frames():
    from sam6d_b200 import synth
    return [synth.make_fastsam_frame(480, 640, s) for s in (0, 1)]


@pytest.fixture(scope="module")
def oracle_out(sd, frames):
    from oracle import fastsam_oracle as fo
    with torch.no_grad():
        return fo.Net(sd).forward(fo.preprocess(frames))


def _run_conv(B, H, W, Cin, Cout, k, s, silu=True, cin_ld=None, c_in0=0, cout_ld=None, c_out0=0, residual=False, tap=None, seed=0):
    from sam6d_b200.fast_sam import YOLOv8Seg, _CW
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    cin_ld, cout_ld = cin_ld or Cin, cout_ld or Cout
    xbuf = torch.randn(B, H, W, cin_ld, device=dev, generator=g).to(torch.bfloat16)
    x = xbuf[..., c_in0:c_in0 + Cin]
    w = (torch.randn(Cout, Cin, k, k, device=dev, generator=g) / (Cin * k * k) ** 0.5).to(torch.bfloat16).float()
    b = torch.randn(Cout, device=dev, generator=g) * 0.1
    cw = _CW(w, b)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    Hy, Wy = (2 * Ho, 2 * Wo) if tap is not None else (Ho, Wo)
    ybuf = torch.full((B, Hy, Wy, cout_ld), 7.0, device=dev, dtype=torch.bfloat16)
    y = ybuf[..., c_out0:c_out0 + Cout]
    rbuf = torch.randn(B, Ho, Wo, cout_ld, device=dev, generator=g).to(torch.bfloat16) if residual else None
    r = rbuf[..., c_out0:c_out0 + Cout] if residual else None
    YOLOv8Seg._conv(x, cw, y, stride=s, silu=silu, res=r, tap=tap)
    torch.cuda.synchronize()
    xf = x.float().permute(0, 3, 1, 2)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    ref = F.conv2d(xf, w, b, s, k // 2)
    mag = F.conv2d(xf.abs(), w.abs(), b.abs(), s, k // 2)
    torch.backends.cudnn.allow_tf32 = prev
    if silu:
        ref = F.silu(ref)
    if residual:
        ref = ref + r.float().permute(0, 3, 1, 2)
        mag = mag + r.float().abs().permute(0, 3, 1, 2)
    ref, mag = ref.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)
    got = y[:, tap[0]::2, tap[1]::2] if tap is not None else y
    # error model: both sides accumulate the K = k*k*Cin products of the same bf16-exact operands in fp32 (each within
    # gamma_K * sum|x w| of the exact sum, gamma_K ~ K u_fp32; SiLU is 1-Lipschitz-ish (|silu'| <= 1.1) and the residual adds
    # exactly), then the kernel rounds once to bf16 (half an ulp: |y| u_bf16 / 2 -- we allow a full u_bf16 for the SiLU evaluation)
    K = k * k * Cin
    bound = 2 * 1.1 * K * U_FP32 * mag + U_BF16 * ref.abs() + 1e-30
    err = (got.float() - ref).abs()
    assert torch.isfinite(got.float()).all()
    assert (err <= bound).all(), f"max err {err.max().item():.3g}, worst err/bound {(err / bound).max().item():.3g}"
    # nothing outside the written slice / taps changed
    if c_out0 or cout_ld != Cout:
        outside = torch.cat([ybuf[..., :c_out0], ybuf[..., c_out0 + Cout:]], -1)
        assert (outside == 7.0).all()
    return (err / bound).max().item()


def _layer_shapes():
    from oracle import fastsam_oracle as fo
    seen = []
    for l in fo.conv_shapes(480, 640):
        key = (l["H"], l["W"], l["Cin"], l["Cout"], l["k"], l["s"])
        if l["Cin"] != 3 and key not in seen:             # the Cin = 3 stem is its own kernel
            seen.append(key)
    return seen


@pytest.mark.parametrize("B", [1, 3])
def test_conv_every_layer_shape(B):
    worst = 0.0
    shapes = _layer_shapes()
    for i, (H, W, Cin, Cout, k, s) in enumerate(shapes):
        worst = max(worst, _run_conv(B, H, W, Cin, Cout, k, s, seed=i))
    print(f"{len(shapes)} distinct layer shapes at B={B}: worst err / bound = {worst:.3f}")


@pytest.mark.parametrize("case", [
    dict(B=2, H=15, W=20, Cin=64, Cout=80, k=3, s=1),
    dict(B=2, H=15, W=20, Cin=64, Cout=80, k=3, s=2),
    dict(B=1, H=1, W=1, Cin=16, Cout=8, k=3, s=1),
    dict(B=1, H=1, W=1, Cin=16, Cout=8, k=3, s=2),
    dict(B=2, H=17, W=33, Cin=24, Cout=136, k=3, s=1),                     # Cin tail in a single partial slab, two N tiles
    dict(B=2, H=30, W=40, Cin=200, Cout=97, k=1, s=1, silu=False),         # Cin tail 200 = 3 x 64 + 8, odd Cout
    dict(B=2, H=30, W=40, Cin=80, Cout=80, k=3, s=1, cin_ld=480, c_in0=400, cout_ld=480, c_out0=80),   # slices, ld > C
    dict(B=2, H=30, W=40, Cin=160, Cout=160, k=3, s=1, cin_ld=640, c_in0=160, cout_ld=640, c_out0=320, residual=True),
    dict(B=2, H=31, W=41, Cin=96, Cout=64, k=3, s=2, cin_ld=104, c_in0=8),
    dict(B=2, H=15, W=20, Cin=320, Cout=320, k=1, s=1, silu=False, tap=(0, 1)),
    dict(B=2, H=15, W=20, Cin=320, Cout=320, k=1, s=1, silu=False, tap=(1, 0)),
])
def test_conv_edge_cases(case):
    _run_conv(**case)


def test_sppf_kernel_matches_cascaded_pools_tensor_args():
    from sam6d_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(3)
    buf = torch.zeros(2, 15, 20, 1280, device="cuda", dtype=torch.bfloat16)
    buf[..., :320] = torch.randn(2, 15, 20, 320, device="cuda", generator=g).to(torch.bfloat16)
    _lib.call("sam6d_yolo_sppf", buf, 1280, 2, 15, 20, 320)
    x = buf[..., :320].float().permute(0, 3, 1, 2)
    y1 = F.max_pool2d(x, 5, 1, 2); y2 = F.max_pool2d(y1, 5, 1, 2); y3 = F.max_pool2d(y2, 5, 1, 2)
    ref = torch.cat((y1, y2, y3), 1).permute(0, 2, 3, 1)
    assert torch.equal(buf[..., 320:].float(), ref)


def _decode_all(head, sizes):
    """GPU decode of every anchor (threshold below any sigmoid) -> (A, 38) rows in anchor order"""
    from sam6d_b200 import _lib
    B, A, _ = head.shape
    cand = torch.empty(B, A, 38, device="cuda")
    count = torch.empty(B, dtype=torch.int32, device="cuda")
    _lib.call("sam6d_yolo_decode", head, head.stride(1), head.stride(0), B, *[v for hw in sizes for v in hw], -1.0, cand, count)
    assert (count.cpu() == A).all()
    return cand


def test_network_matches_oracle_tensor_args(sd, frames, oracle_out):
    """whole network, two frames in one batch, bf16 activations vs the fp32 oracle.  Error model: every layer rounds its output
    to bf16 once (relative u_bf16 = 2^-8 at most, ~2^-10 rms); about 60 such roundings lie on the longest path and the seeded
    layers neither amplify nor damp much (activations stay O(1)), so the errors add up like a random walk to ~sqrt(60) x 2^-10
    ~ 1 % of an output's spread; the bound is 5 % of the spread (rms) -- 5x headroom -- for every compared output."""
    from oracle import fastsam_oracle as fo
    from sam6d_b200.fast_sam import YOLOv8Seg
    net = YOLOv8Seg().cuda().eval()
    net.load_state_dict(sd, strict=True)
    head, proto = net(torch.from_numpy(np.stack(frames)).cuda())
    torch.cuda.synchronize()
    sizes = oracle_out["sizes"]
    rows = _decode_all(head, sizes).cpu()
    pred = oracle_out["pred"]
    ref_box = fo.xywh2xyxy(pred[:, :4].transpose(1, 2))
    ref_score = pred[:, 4]
    ref_mc = pred[:, 5:].transpose(1, 2)
    ref_proto = oracle_out["proto"].permute(0, 2, 3, 1)

    def rel(a, b):
        return ((a - b).norm() / (b - b.mean()).norm()).item()

    r = dict(boxes=rel(rows[..., :4], ref_box), scores=rel(rows[..., 4], ref_score), coeffs=rel(rows[..., 6:], ref_mc),
             proto=rel(proto.cpu(), ref_proto))
    print("rms error / rms spread:", {k: f"{v:.4f}" for k, v in r.items()})
    assert all(v < 0.05 for v in r.values()), r


def _anchor_of(rows_mc, raw_mc):
    """anchor index of each kept row, found by its coefficients (copied bit for bit from the head row)"""
    idx = []
    for m in rows_mc:
        hit = torch.nonzero((raw_mc == m).all(1)).flatten()
        assert hit.numel() == 1
        idx.append(hit.item())
    return idx


def test_postprocess_exact_on_oracle_head(sd, oracle_out):
    """decode -> stable sort -> NMS -> max_det -> masks on the GPU from the oracle's own head and proto: the discrete decisions
    must be the oracle's, after checking that no score or IoU sits within 1e-5 of the 0.25 / 0.9 thresholds"""
    import torchvision
    from oracle import fastsam_oracle as fo
    from sam6d_b200.fast_sam import FastSAM
    seg = FastSAM(None)
    for b in range(2):
        pred = oracle_out["pred"][b:b + 1]
        score = pred[0, 4]
        assert (score - 0.25).abs().min() > 1e-5
        cand = fo.xywh2xyxy(pred[0, :4].t()[score > 0.25])
        iou = torchvision.ops.box_iou(cand, cand).fill_diagonal_(0)
        assert (iou - 0.9).abs().min() > 1e-5
        det = fo.non_max_suppression(pred)[0]
        assert det.shape[0] == 200 and (score > 0.25).sum() > 200              # the max_det cut is hit
        ref_masks, prob = fo.process_mask(oracle_out["proto"][b], det[:, 6:], det[:, :4], (480, 640), return_prob=True)
        head = oracle_out["raw"][b].cuda()
        proto = oracle_out["proto"][b].permute(1, 2, 0).contiguous().cuda()
        out = seg.postprocess(head, proto, (480, 640))
        rows = out["rows"].cpu()
        raw_mc = oracle_out["raw"][b][:, 65:]
        assert _anchor_of(rows[:, 6:], raw_mc) == _anchor_of(det[:, 6:], raw_mc)
        torch.testing.assert_close(rows[:, :4], det[:, :4], rtol=4 * 2.0 ** -23, atol=1e-4)
        torch.testing.assert_close(rows[:, 4], det[:, 4], rtol=4 * 2.0 ** -23, atol=0)
        near = (prob - 0.5).abs() < 1e-5
        diff = out["masks"].cpu().bool() != ref_masks.bool()
        print(f"frame {b}: {det.shape[0]} kept, {near.sum().item()} mask pixels within 1e-5 of 0.5, {diff.sum().item()} differ")
        assert not (diff & ~near).any()


def _mask_iou(a, b):
    a, b = a.flatten(1).float(), b.flatten(1).float()
    inter = a @ b.t()
    union = a.sum(1)[:, None] + b.sum(1)[None, :] - inter
    return torch.where(union > 0, inter / union.clamp(min=1), torch.ones_like(inter))


@pytest.mark.parametrize("hw", [(480, 640), (720, 1280)])
def test_generate_masks_end_to_end(sd, hw):
    from oracle import fastsam_oracle as fo
    from sam6d_b200 import synth
    from sam6d_b200.fast_sam import FastSAM
    img = synth.make_fastsam_frame(*hw, seed=5)
    seg = FastSAM(None, dict(iou_threshold=0.9, conf_threshold=0.05, max_det=200))
    seg.model.load_state_dict(sd, strict=True)
    a = seg.generate_masks(img)
    b = seg.generate_masks(img)
    assert torch.equal(a["masks"], b["masks"]) and torch.equal(a["boxes"], b["boxes"])
    assert a["masks"].shape[1:] == hw and a["masks"].dtype == torch.float32 and a["boxes"].shape == (a["masks"].shape[0], 4)
    ref = fo.generate_masks(sd, img)
    iou = _mask_iou(ref["masks"] > 0.5, a["masks"].cpu() > 0.5)
    matched = (iou.amax(1) >= 0.9).float().mean().item()
    print(f"{hw}: oracle {ref['masks'].shape[0]} detections, GPU {a['masks'].shape[0]}, matched at mask IoU >= 0.9: {matched:.3f}")
    assert matched >= 0.9


def test_ism_fastsam_cli_then_pem_cli(tmp_path, golden_dir):
    """the reference demo with SEGMENTOR_MODEL=fastsam: templates -> ISM CLI (FastSAM proposals, DINOv2 descriptors, scores ->
    detection_ism.json) -> PEM CLI consuming that file.  Seeded weights: record format and validity are checked."""
    import cv2
    from scipy.spatial import ConvexHull
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, pem_run_inference_custom as pem_cli, render_point_templates as rpt
    from test_gpu_cli import _write_ply
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
    assert ism_cli.main(common + ["--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1"]) == 0
    dets = json.load(open(os.path.join(out, "sam6d_results", "detection_ism.json")))
    print(f"ISM CLI (fastsam): {len(dets)} detections")
    assert len(dets) >= 1
    for d in dets:
        assert set(["scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation"]) <= set(d)
        assert d["segmentation"]["size"] == [480, 640] and sum(d["segmentation"]["counts"]) == 480 * 640
        assert np.isfinite(d["score"])
    np.random.seed(0)
    assert pem_cli.main(common + ["--seg_path", os.path.join(out, "sam6d_results", "detection_ism.json"), "--random_weights",
                                  "--det_score_thresh", "-1"]) == 0
    res = json.load(open(os.path.join(out, "sam6d_results", "detection_pem.json")))
    assert len(res) <= len(dets)
    for r in res:
        R = np.array(r["R"])
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-4) and np.isfinite(np.array(r["t"])).all()
