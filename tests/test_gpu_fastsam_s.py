"""GPU: FastSAM-s (YOLOv8s-seg) on sm_90a.  The s network, post-processing and CLIs against the fp32 CPU restatement
oracle/fastsam_oracle.py on seeded weights (synth.make_fastsam_state_dict(scale="s")); every convolution shape of s and the
narrow-channel edge cases of its layers (Cout <= 64 in one 128-wide N tile) against fp64; the stem at 32 channels."""
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
    return synth.make_fastsam_state_dict(1, scale="s")


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
    """one sam6d_conv2d_tc launch against the fp64 convolution of the same bf16 operands; the bound of
    test_gpu_fastsam._run_conv: 2 x 1.1 x K u_fp32 x sum|x w| for the two fp32 accumulations (SiLU's slope <= 1.1) plus one
    bf16 rounding (a full u_bf16 for the SiLU evaluation)"""
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
    rbuf = torch.randn(B, Hy, Wy, cout_ld, device=dev, generator=g).to(torch.bfloat16) if residual else None
    r = rbuf[..., c_out0:c_out0 + Cout] if residual else None
    YOLOv8Seg._conv(x, cw, y, stride=s, silu=silu, res=r, tap=tap)
    torch.cuda.synchronize()
    xd, wd, bd = x.double().permute(0, 3, 1, 2), w.double(), b.double()
    ref = F.conv2d(xd, wd, bd, s, k // 2)
    mag = F.conv2d(xd.abs(), wd.abs(), bd.abs(), s, k // 2)
    if silu:
        ref = F.silu(ref)
    ref, mag = ref.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)
    got = y[:, tap[0]::2, tap[1]::2] if tap is not None else y
    if residual:
        rr = r[:, tap[0]::2, tap[1]::2] if tap is not None else r
        ref, mag = ref + rr.double(), mag + rr.double().abs()
    K = k * k * Cin
    bound = 2 * 1.1 * K * U_FP32 * mag + U_BF16 * ref.abs() + 1e-30
    err = (got.double() - ref).abs()
    assert torch.isfinite(got.float()).all()
    assert (err <= bound).all(), f"max err {err.max().item():.3g}, worst err/bound {(err / bound).max().item():.3g}"
    untouched = ybuf.clone()
    if tap is not None:
        untouched[:, tap[0]::2, tap[1]::2, c_out0:c_out0 + Cout] = 7.0
    else:
        untouched[..., c_out0:c_out0 + Cout] = 7.0
    assert (untouched == 7.0).all(), "a pixel or channel outside the output slice / tap was written"
    return (err / bound).max().item()


def _s_layer_shapes():
    from sam6d_b200.fast_sam import conv_shapes
    seen = []
    for l in conv_shapes("s", 480, 640):
        key = (l["H"], l["W"], l["Cin"], l["Cout"], l["k"], l["s"])
        if l["Cin"] != 3 and "upsample" not in l["name"] and key not in seen:
            seen.append(key)
    return seen


@pytest.mark.parametrize("B", [1, 3])
def test_conv_every_s_layer_shape(B):
    shapes = _s_layer_shapes()
    worst = max(_run_conv(B, H, W, Cin, Cout, k, s, seed=i) for i, (H, W, Cin, Cout, k, s) in enumerate(shapes))
    print(f"{len(shapes)} distinct FastSAM-s layer shapes at B={B}: worst err / bound = {worst:.3f}")


@pytest.mark.parametrize("case", [
    dict(B=2, H=15, W=20, Cin=64, Cout=8, k=3, s=1),
    dict(B=2, H=15, W=20, Cin=32, Cout=24, k=3, s=1),
    dict(B=2, H=15, W=20, Cin=64, Cout=40, k=1, s=1),
    dict(B=2, H=15, W=20, Cin=96, Cout=48, k=3, s=1),
    dict(B=2, H=15, W=20, Cin=128, Cout=64, k=3, s=1),
    dict(B=2, H=17, W=33, Cin=40, Cout=33, k=3, s=1, silu=False),            # odd Cout, Cin tail
    dict(B=2, H=30, W=40, Cin=224, Cout=97, k=1, s=1, silu=False),           # the s head's last layer
    dict(B=2, H=17, W=33, Cin=24, Cout=136, k=3, s=1),                       # two N tiles, the last ragged
    dict(B=2, H=30, W=40, Cin=32, Cout=32, k=3, s=1, cin_ld=96, c_in0=64, cout_ld=96, c_out0=32),       # slices, ld > C
    dict(B=2, H=30, W=40, Cin=64, Cout=64, k=3, s=1, cin_ld=256, c_in0=64, cout_ld=256, c_out0=128, residual=True),
    dict(B=2, H=31, W=41, Cin=32, Cout=64, k=3, s=2),
    dict(B=2, H=31, W=41, Cin=64, Cout=48, k=3, s=2, cin_ld=104, c_in0=8),
    dict(B=2, H=15, W=20, Cin=128, Cout=128, k=1, s=1, silu=False, tap=(0, 1)),
    dict(B=2, H=15, W=20, Cin=128, Cout=128, k=1, s=1, silu=False, tap=(1, 1)),
    dict(B=1, H=1, W=1, Cin=16, Cout=8, k=3, s=1),
    dict(B=1, H=1, W=1, Cin=32, Cout=64, k=3, s=2),
])
def test_conv_narrow_channel_edge_cases(case):
    _run_conv(**case)


def test_conv_fp32_output_32_channels():
    """Proto.cv3 of s: 128 -> 32, SiLU, fp32 out"""
    from sam6d_b200.fast_sam import YOLOv8Seg, _CW
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(2, 24, 32, 128, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(32, 128, 1, 1, device="cuda", generator=g) / 128 ** 0.5).to(torch.bfloat16).float()
    b = torch.randn(32, device="cuda", generator=g) * 0.1
    y = torch.full((2, 24, 32, 32), 7.0, device="cuda")
    YOLOv8Seg._conv(x, _CW(w, b), y)
    ref = F.silu(F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double())).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs().permute(0, 3, 1, 2), w.double().abs(), b.double().abs()).permute(0, 2, 3, 1)
    bound = 2 * 1.1 * 128 * U_FP32 * mag + 1e-30              # fp32 out: no bf16 rounding
    assert ((y.double() - ref).abs() <= bound).all()


def test_stem_32_channels_matches_fp64_tensor_args():
    from sam6d_b200 import _lib
    g = torch.Generator().manual_seed(2)
    img = np.random.RandomState(3).randint(0, 256, (2, 33, 47, 3)).astype(np.uint8)    # odd sizes: the ceil(H/2) border
    w = torch.randn(32, 3, 3, 3, generator=g) * 0.5
    b = torch.randn(32, generator=g) * 0.1
    out = torch.full((2, 17, 24, 32), 7.0, device="cuda", dtype=torch.bfloat16)
    frames = torch.from_numpy(img).cuda()
    w_dev, b_dev = w.permute(0, 2, 3, 1).contiguous().cuda(), b.cuda()          # (out, ky, kx, in); kept alive over the launch
    _lib.call("sam6d_yolo_stem_c", frames, 2, 33, 47, 32, w_dev, b_dev, out)
    torch.cuda.synchronize()
    x = torch.from_numpy(np.ascontiguousarray(img[..., ::-1])).double().permute(0, 3, 1, 2) / 255.0
    pre = F.conv2d(x, w.double(), b.double(), 2, 1)
    ref = F.silu(pre).permute(0, 2, 3, 1)
    mag = F.conv2d(x.abs(), w.double().abs(), b.double().abs(), 2, 1).permute(0, 2, 3, 1)
    # 27 fp32 fmas (gamma_27 u_fp32 x sum|x w|, /255 rounded once more), SiLU with expf (a few ulp), one bf16 rounding
    bound = 1.1 * 30 * U_FP32 * mag + 4 * U_FP32 * ref.abs() + U_BF16 * ref.abs() + 1e-30
    err = (out.cpu().double() - ref).abs()
    assert (err <= bound).all(), f"worst err/bound {(err / bound).max().item():.3g}"


def test_stem_rejects_bad_width_tensor_args():
    from sam6d_b200 import _lib
    img = torch.zeros(1, 4, 4, 3, dtype=torch.uint8, device="cuda")
    w, b = torch.zeros(40, 27, device="cuda"), torch.zeros(40, device="cuda")
    out = torch.zeros(1, 2, 2, 40, device="cuda", dtype=torch.bfloat16)
    for C in (40, 96):
        with pytest.raises(_lib.Sam6dError, match="invalid argument"):
            _lib.call("sam6d_yolo_stem_c", img, 1, 4, 4, C, w, b, out)


def _decode_all(head, sizes):
    from test_gpu_fastsam import _decode_all as d
    return d(head, sizes)


def test_s_network_matches_oracle_tensor_args(sd, frames, oracle_out):
    """whole s network, two frames in one batch, bf16 activations vs the fp32 oracle; the error model of
    test_gpu_fastsam.test_network_matches_oracle_tensor_args (s has fewer layers on its longest path than x): 5 % of the rms spread"""
    from oracle import fastsam_oracle as fo
    from sam6d_b200.fast_sam import YOLOv8Seg
    net = YOLOv8Seg("s").cuda().eval()
    net.load_state_dict(sd, strict=True)
    head, proto = net(torch.from_numpy(np.stack(frames)).cuda())
    torch.cuda.synchronize()
    rows = _decode_all(head, oracle_out["sizes"]).cpu()
    pred = oracle_out["pred"]

    def rel(a, b):
        return ((a - b).norm() / (b - b.mean()).norm()).item()

    r = dict(boxes=rel(rows[..., :4], fo.xywh2xyxy(pred[:, :4].transpose(1, 2))), scores=rel(rows[..., 4], pred[:, 4]),
             coeffs=rel(rows[..., 6:], pred[:, 5:].transpose(1, 2)), proto=rel(proto.cpu(), oracle_out["proto"].permute(0, 2, 3, 1)))
    print("rms error / rms spread:", {k: f"{v:.4f}" for k, v in r.items()})
    assert all(v < 0.05 for v in r.values()), r


def test_s_postprocess_exact_on_oracle_head(sd, oracle_out):
    """decode -> stable sort -> NMS -> max_det -> masks from the oracle's own s head and proto: the oracle's decisions exactly"""
    import torchvision
    from oracle import fastsam_oracle as fo
    from sam6d_b200.fast_sam import FastSAM
    from test_gpu_fastsam import _anchor_of
    seg = FastSAM(None, scale="s")
    for b in range(2):
        pred = oracle_out["pred"][b:b + 1]
        score = pred[0, 4]
        assert (score - 0.25).abs().min() > 1e-5
        cand = fo.xywh2xyxy(pred[0, :4].t()[score > 0.25])
        iou = torchvision.ops.box_iou(cand, cand).fill_diagonal_(0)
        assert (iou - 0.9).abs().min() > 1e-5
        det = fo.non_max_suppression(pred)[0]
        assert det.shape[0] == 200 and (score > 0.25).sum() > 200
        ref_masks, prob = fo.process_mask(oracle_out["proto"][b], det[:, 6:], det[:, :4], (480, 640), return_prob=True)
        out = seg.postprocess(oracle_out["raw"][b].cuda(), oracle_out["proto"][b].permute(1, 2, 0).contiguous().cuda(), (480, 640))
        rows = out["rows"].cpu()
        raw_mc = oracle_out["raw"][b][:, 65:]
        assert _anchor_of(rows[:, 6:], raw_mc) == _anchor_of(det[:, 6:], raw_mc)
        torch.testing.assert_close(rows[:, :4], det[:, :4], rtol=4 * 2.0 ** -23, atol=1e-4)
        torch.testing.assert_close(rows[:, 4], det[:, 4], rtol=4 * 2.0 ** -23, atol=0)
        near = (prob - 0.5).abs() < 1e-5
        diff = out["masks"].cpu().bool() != ref_masks.bool()
        print(f"frame {b}: {det.shape[0]} kept, {int(ref_masks.sum())} mask pixels set, {near.sum().item()} within 1e-5 of 0.5, {diff.sum().item()} differ")
        assert ref_masks.sum() > 0 and not (diff & ~near).any()


@pytest.mark.parametrize("hw", [(480, 640), (720, 1280)])
def test_s_generate_masks_end_to_end(sd, hw):
    from oracle import fastsam_oracle as fo
    from sam6d_b200 import synth
    from sam6d_b200.fast_sam import FastSAM
    from test_gpu_fastsam import _mask_iou
    img = synth.make_fastsam_frame(*hw, seed=5)
    seg = FastSAM(None, dict(iou_threshold=0.9, conf_threshold=0.05, max_det=200), scale="s")
    seg.model.load_state_dict(sd, strict=True)
    a = seg.generate_masks(img)
    b = seg.generate_masks(img)
    assert torch.equal(a["masks"], b["masks"]) and torch.equal(a["boxes"], b["boxes"])
    assert a["masks"].shape[1:] == hw and a["masks"].dtype == torch.float32 and a["boxes"].shape == (a["masks"].shape[0], 4)
    ref = fo.generate_masks(sd, img)
    iou = _mask_iou(ref["masks"] > 0.5, a["masks"].cpu() > 0.5)
    matched = (iou.amax(1) >= 0.9).float().mean().item()
    print(f"{hw}: oracle {ref['masks'].shape[0]} detections, GPU {a['masks'].shape[0]}, matched at mask IoU >= 0.9: {matched:.3f}")
    assert ref["masks"].shape[0] >= 1 and matched >= 0.9


def test_ism_cli_fastsam_s_then_pem_cli_and_sam6d_frame(tmp_path, golden_dir):
    """--fastsam_model FastSAM-s through the ISM and PEM CLIs, then one SAM6D(fastsam_model="FastSAM-s") frame giving the same
    records (seeded weights)"""
    from sam6d_b200.pipeline import SAM6D
    from test_gpu_pipeline import _chain, _example, _frame_inputs, _same_records
    out = str(tmp_path)
    gold, cad, common = _example(out, golden_dir)
    ism_ref, pem_ref = _chain(out, cad, common, dict(ism=["--segmentor_model", "fastsam", "--fastsam_model", "FastSAM-s"]))
    print(f"FastSAM-s: chained CLIs {len(ism_ref)} ISM / {len(pem_ref)} PEM records")
    assert len(ism_ref) >= 1 and len(pem_ref) >= 1
    for d in ism_ref:
        assert d["segmentation"]["size"] == [480, 640] and sum(d["segmentation"]["counts"]) == 480 * 640 and np.isfinite(d["score"])
    for r in pem_ref:
        R = np.array(r["R"])
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-4) and np.isfinite(np.array(r["t"])).all()
    model = SAM6D(segmentor="fastsam", fastsam_model="FastSAM-s", random_weights=True, confidence_thresh=-1, det_score_thresh=-1)
    assert model.seg.model.scale == "s"
    rng = np.random.RandomState(0)
    obj = model.onboard(cad, template_size=192, rng=rng)
    res = model(*_frame_inputs(gold), obj, rng=rng)
    _same_records(ism_ref, json.loads(json.dumps(res.ism)), "FastSAM-s ISM")
    _same_records(pem_ref, json.loads(json.dumps(res.pem)), "FastSAM-s PEM")
