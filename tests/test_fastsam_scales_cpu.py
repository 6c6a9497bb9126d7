"""CPU: FastSAM at its two published scales (sam6d_b200/fast_sam.py): the x and s layer tables, the checkpoint loader's scale
inference and rejection of other layouts, FastSAM's scale keyword, the seeded weights of both scales, and --fastsam_model."""
import sys

import pytest
import torch


def _params(m):
    return sum(p.numel() for p in m.parameters())


def test_scale_layouts_and_parameter_counts():
    from sam6d_b200.fast_sam import YOLOv8Seg, scale_layout
    x, s = YOLOv8Seg("x"), YOLOv8Seg("s")
    assert _params(YOLOv8Seg()) == _params(x) == 71_751_811
    assert list(YOLOv8Seg().state_dict()) == list(x.state_dict())
    assert _params(s) == 11_790_483
    sd = s.state_dict()
    for k, shape in (("model.0.conv.weight", (32, 3, 3, 3)), ("model.2.cv2.conv.weight", (64, 96, 1, 1)),
                     ("model.9.cv2.conv.weight", (512, 1024, 1, 1)), ("model.22.cv4.0.0.conv.weight", (32, 128, 3, 3)),
                     ("model.22.proto.upsample.weight", (128, 128, 2, 2)), ("model.22.proto.cv3.conv.weight", (32, 128, 1, 1)),
                     ("model.22.cv2.0.0.conv.weight", (64, 128, 3, 3)), ("model.22.cv3.0.0.conv.weight", (128, 128, 3, 3))):
        assert tuple(sd[k].shape) == shape, k
    lay = scale_layout("s")
    assert lay.c == (32, 64, 128, 256, 512) and (lay.n3, lay.n6, lay.npr) == (1, 2, 128)
    for i, n in ((2, 1), (4, 2), (6, 2), (8, 1), (12, 1), (15, 1), (18, 1), (21, 1)):
        assert len(s.model[i].m) == n
    with pytest.raises(ValueError, match="scale"):
        YOLOv8Seg("n")


def test_parameter_counts_at_80_classes():
    """the same rules at nc = 80 give ultralytics' published 11.8 M (YOLOv8s-seg) and 71.8 M (YOLOv8x-seg)"""
    from sam6d_b200.fast_sam import Segment, YOLOv8Seg, scale_layout
    for scale, want in (("s", 11_821_056), ("x", 71_827_888)):
        m, lay = YOLOv8Seg(scale), scale_layout(scale)
        c = lay.c
        m.model[22] = Segment(nc=80, npr=lay.npr, ch=(c[2], c[3], c[4]))
        assert _params(m) == want, scale


def test_conv_shapes_follow_the_layer_table():
    from sam6d_b200.fast_sam import conv_shapes
    from oracle import fastsam_oracle as fo
    x = conv_shapes("x", 480, 640)
    ref = {l["name"]: l for l in fo.conv_shapes(480, 640)}
    for l in x:
        if l["name"] in ref:
            assert {k: l[k] for k in ("Cin", "Cout", "k", "s", "H", "W")} == {k: ref[l["name"]][k] for k in ("Cin", "Cout", "k", "s", "H", "W")}
    s = {l["name"]: l for l in conv_shapes("s", 480, 640)}
    assert (s["model.2.cv2"]["Cin"], s["model.2.cv2"]["Cout"]) == (96, 64)
    assert (s["model.22.head.0.first"]["Cout"], s["model.22.head.0.last"]["Cin"]) == (224, 224)
    assert (s["model.9.cv1"]["Cout"], s["model.9.cv2"]["Cin"]) == (256, 1024)


# ---------------------------------------------------------------------------------------------------------------- loader
def _save_fake(path, net):
    from test_fastsam_cpu import _fake_ultralytics_checkpoint
    import sam6d_b200.fast_sam as fs
    orig = fs.YOLOv8Seg
    try:
        fs.YOLOv8Seg = lambda: net                                  # the helper builds YOLOv8Seg(); hand it this network
        return _fake_ultralytics_checkpoint(path)
    finally:
        fs.YOLOv8Seg = orig


def test_loader_infers_s_from_ultralytics_pickle(tmp_path):
    from sam6d_b200.fast_sam import YOLOv8Seg, checkpoint_scale, load_fastsam_checkpoint
    path = str(tmp_path / "FastSAM-s.pt")
    ref = _save_fake(path, YOLOv8Seg("s"))
    assert "ultralytics" not in sys.modules
    sd = load_fastsam_checkpoint(path)
    assert set(sd) == set(ref) and all(torch.equal(sd[k], ref[k]) for k in sd)
    assert checkpoint_scale(sd) == "s"
    YOLOv8Seg("s").load_state_dict(sd, strict=True)


def _n_shaped():
    """YOLOv8n-seg's layout (depth 0.33, width 0.25): widths 16 / 32 / 64 / 128 / 256"""
    from sam6d_b200.fast_sam import C2f, Conv, SPPF, Segment, YOLOv8Seg, _Layer
    net = YOLOv8Seg("s")
    c0, c1, c2, c3, c4 = 16, 32, 64, 128, 256
    L = [Conv(3, c0, 3, 2), Conv(c0, c1, 3, 2), C2f(c1, c1, 1, True), Conv(c1, c2, 3, 2), C2f(c2, c2, 2, True),
         Conv(c2, c3, 3, 2), C2f(c3, c3, 2, True), Conv(c3, c4, 3, 2), C2f(c4, c4, 1, True), SPPF(c4, c4),
         _Layer(), _Layer(), C2f(c4 + c3, c3, 1, False), _Layer(), _Layer(), C2f(c3 + c2, c2, 1, False),
         Conv(c2, c2, 3, 2), _Layer(), C2f(c2 + c3, c3, 1, False), Conv(c3, c3, 3, 2), _Layer(), C2f(c3 + c4, c4, 1, False),
         Segment(npr=64, ch=(c2, c3, c4))]
    net.model = torch.nn.ModuleList(L)
    return net


def test_loader_rejects_other_scales_naming_what_it_found(tmp_path):
    from sam6d_b200.fast_sam import load_fastsam_checkpoint
    path = str(tmp_path / "FastSAM-n.pt")
    _save_fake(path, _n_shaped())
    with pytest.raises(ValueError, match=r"not a YOLOv8x-seg or YOLOv8s-seg .*found stem width 16, SPPF width 256, C2f depths 1 / 2"):
        load_fastsam_checkpoint(path)


def test_loader_rejects_a_damaged_s_checkpoint(tmp_path):
    from sam6d_b200.fast_sam import YOLOv8Seg, load_fastsam_checkpoint
    net = YOLOv8Seg("s")
    net.model[22].proto.cv3 = type(net.model[22].proto.cv2)(128, 16)
    path = str(tmp_path / "bad-s.pt")
    _save_fake(path, net)
    with pytest.raises(ValueError, match=r"not a YOLOv8s-seg .*mis-shaped .*model.22.proto.cv3.conv.weight"):
        load_fastsam_checkpoint(path)


def test_fastsam_scale_keyword(tmp_path):
    from sam6d_b200.fast_sam import FastSAM, YOLOv8Seg
    path = str(tmp_path / "FastSAM-s.pt")
    _save_fake(path, YOLOv8Seg("s"))
    assert FastSAM(path, device="cpu").model.scale == "s"           # the reference's drop-in: checkpoint_path only
    assert FastSAM(path, device="cpu", scale="s").model.scale == "s"
    with pytest.raises(ValueError, match="holds YOLOv8s-seg"):
        FastSAM(path, device="cpu", scale="x")
    assert FastSAM(None, device="cpu").model.scale == "x"
    assert FastSAM(None, device="cpu", scale="s").model.scale == "s"


# ---------------------------------------------------------------------------------------------------------------- seeded weights
# the first values of a few tensors of make_fastsam_state_dict(1) as drawn before the function took a scale
_X_DRAW = {
    "model.0.conv.weight": [-0.36700132489204407, -0.18047772347927094, -0.15732336044311523],
    "model.8.m.2.cv2.bn.running_var": [1.1905808448791504, 0.7234212756156921, 0.5438820123672485],
    "model.22.cv4.2.2.weight": [-4.967733860015869, 40.98596954345703, 1.1817657947540283],
    "model.22.proto.upsample.bias": [-0.007349352817982435, 0.007905598729848862, -0.0030178099405020475],
}


def test_seeded_x_draw_unchanged():
    """existing tests and CLI runs rely on the x draw"""
    from sam6d_b200 import synth
    sd = synth.make_fastsam_state_dict(1)
    sd2 = synth.make_fastsam_state_dict(1, scale="x")
    assert list(sd) == list(sd2) and all(torch.equal(sd[k], sd2[k]) for k in sd)
    for k, v in _X_DRAW.items():
        assert torch.equal(sd[k].flatten()[:3], torch.tensor(v, dtype=torch.float32)), k
    assert (sd["model.22.cv3.0.2.bias"] == 0).all() and (sd["model.22.cv4.1.2.bias"] == 0.065).all()


def test_seeded_s_weights_properties_on_oracle():
    """make_fastsam_state_dict(scale="s") on the two test frames of the GPU tests: several hundred anchors pass conf 0.25, more
    than max_det = 200 survive NMS, no score within 1e-5 of 0.25 and no candidate IoU within 1e-5 of 0.9 (so the GPU
    post-processing must reach the oracle's decisions exactly), and the kept masks are not empty"""
    import torchvision
    from oracle import fastsam_oracle as fo
    from sam6d_b200 import synth
    sd = synth.make_fastsam_state_dict(1, scale="s")
    assert fo.param_count(sd) == 11_790_483
    frames = [synth.make_fastsam_frame(480, 640, s) for s in (0, 1)]
    with torch.no_grad():
        out = fo.Net(sd).forward(fo.preprocess(frames))
    assert out["pred"].shape == (2, 37, 6300) and out["proto"].shape == (2, 32, 120, 160)
    for b in range(2):
        pred = out["pred"][b:b + 1]
        score = pred[0, 4]
        n_pass = int((score > 0.25).sum())
        kept = fo.non_max_suppression(pred, max_det=10 ** 6)[0]
        print(f"frame {b}: {n_pass} pass conf 0.25, {kept.shape[0]} survive NMS")
        assert 250 <= n_pass <= 2000 and kept.shape[0] > 200
        assert (score - 0.25).abs().min() > 1e-5
        cand = fo.xywh2xyxy(pred[0, :4].t()[score > 0.25])
        assert (torchvision.ops.box_iou(cand, cand).fill_diagonal_(0) - 0.9).abs().min() > 1e-5
        masks = fo.process_mask(out["proto"][b], kept[:200, 6:], kept[:200, :4], (480, 640))
        assert (masks.flatten(1).sum(1) > 0).float().mean() > 0.5


# ---------------------------------------------------------------------------------------------------------------- CLIs
def test_cli_accepts_fastsam_model():
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, run_sam6d
    ap = ism_cli.get_parser()
    assert ap.parse_args([]).fastsam_model == "FastSAM-x"
    assert ap.parse_args(["--segmentor_model", "fastsam", "--fastsam_model", "FastSAM-s"]).fastsam_model == "FastSAM-s"
    with pytest.raises(SystemExit):
        ap.parse_args(["--fastsam_model", "FastSAM-n"])
    req = ["--output_dir", "o", "--cad_path", "c.ply", "--rgb_path", "r.png", "--depth_path", "d.png", "--cam_path", "k.json"]
    assert run_sam6d.get_parser().parse_args(req).fastsam_model == "FastSAM-x"
    assert run_sam6d.get_parser().parse_args(req + ["--fastsam_model", "FastSAM-s"]).fastsam_model == "FastSAM-s"


def test_sam6d_rejects_unknown_fastsam_model():
    from sam6d_b200.pipeline import SAM6D
    with pytest.raises(ValueError, match="fastsam_model"):
        SAM6D(segmentor="fastsam", fastsam_model="FastSAM-m")
