"""CPU: the FastSAM segmentor's layer table, checkpoint loader, letterbox / scale_boxes geometry, the cascaded-max-pool identity
of SPPF and the CLI surface (sam6d_b200/fast_sam.py, oracle/fastsam_oracle.py)."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F


def test_layer_table_parameter_count_and_keys():
    from sam6d_b200.fast_sam import YOLOv8Seg
    m = YOLOv8Seg()
    assert sum(p.numel() for p in m.parameters()) == 71_751_811
    sd = m.state_dict()
    for k, shape in (("model.0.conv.weight", (80, 3, 3, 3)), ("model.2.cv1.conv.weight", (160, 160, 1, 1)),
                     ("model.2.m.0.cv1.conv.weight", (80, 80, 3, 3)), ("model.9.cv1.conv.weight", (320, 640, 1, 1)),
                     ("model.9.cv2.conv.weight", (640, 1280, 1, 1)), ("model.22.cv2.0.0.conv.weight", (80, 320, 3, 3)),
                     ("model.22.cv3.0.0.conv.weight", (320, 320, 3, 3)), ("model.22.cv3.2.2.weight", (1, 320, 1, 1)),
                     ("model.22.cv4.2.2.weight", (32, 80, 1, 1)), ("model.22.dfl.conv.weight", (1, 16, 1, 1)),
                     ("model.22.proto.upsample.weight", (320, 320, 2, 2)), ("model.22.proto.upsample.bias", (320,)),
                     ("model.22.proto.cv3.conv.weight", (32, 320, 1, 1))):
        assert tuple(sd[k].shape) == shape, k
    for s in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
        assert f"model.0.bn.{s}" in sd
    assert m.model[0].bn.eps == 1e-3


def test_oracle_output_shapes_480x640():
    from oracle import fastsam_oracle as fo
    from sam6d_b200 import synth
    sd = synth.make_fastsam_state_dict(1)
    assert fo.param_count(sd) == 71_751_811
    with torch.no_grad():
        out = fo.Net(sd).forward(torch.rand(1, 3, 480, 640))
    assert out["pred"].shape == (1, 4 + 1 + 32, 6300) and out["proto"].shape == (1, 32, 120, 160)
    assert abs(fo.flops((480, 640)) - 246) < 1


# ---------------------------------------------------------------------------------------------------------------- loader
def _fake_ultralytics_checkpoint(path, half=True, ema=False, extra=None):
    """an ultralytics-style pickle: module classes named ultralytics.* exist only while saving"""
    from sam6d_b200.fast_sam import YOLOv8Seg
    net = YOLOv8Seg()
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(torch.randn_like(p))
    names = ["ultralytics", "ultralytics.nn", "ultralytics.nn.tasks", "ultralytics.nn.modules", "ultralytics.nn.modules.block",
             "ultralytics.nn.modules.conv", "ultralytics.nn.modules.head"]
    mods = {n: types.ModuleType(n) for n in names}
    saved = {n: sys.modules.get(n) for n in names}
    where = {"Conv": "conv", "_Layer": "conv", "Bottleneck": "block", "C2f": "block", "SPPF": "block", "Proto": "block", "DFL": "block",
             "Segment": "head"}
    try:
        sys.modules.update(mods)
        classes = {}
        for sub in net.modules():
            name = type(sub).__name__
            if type(sub).__module__ != "sam6d_b200.fast_sam":
                continue
            if name == "YOLOv8Seg":
                mod, name = "ultralytics.nn.tasks", "SegmentationModel"
            else:
                mod = "ultralytics.nn.modules." + where[name]
                name = "Concat" if name == "_Layer" else name
            if (mod, name) not in classes:
                classes[(mod, name)] = type(name, (nn.Module,), {"__module__": mod})
                setattr(mods[mod], name, classes[(mod, name)])
            sub.__class__ = classes[(mod, name)]
        del net._packed
        model = net.half() if half else net
        ck = {"model": model, "ema": model if ema else None, "epoch": -1, "date": "2023-06-01"}
        if extra:
            ck.update(extra)
        torch.save(ck, path)
        return {k: v.float() for k, v in model.state_dict().items()}
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m


@pytest.mark.parametrize("half,ema", [(True, False), (True, True), (False, False)])
def test_loader_reads_ultralytics_pickle(tmp_path, half, ema):
    from sam6d_b200.fast_sam import YOLOv8Seg, load_fastsam_checkpoint
    path = str(tmp_path / "FastSAM-x.pt")
    ref = _fake_ultralytics_checkpoint(path, half=half, ema=ema)
    assert "ultralytics" not in sys.modules
    sd = load_fastsam_checkpoint(path)
    assert set(sd) == set(ref)
    assert all(torch.equal(sd[k], ref[k]) for k in sd)
    assert all(v.dtype == torch.float32 for k, v in sd.items() if not k.endswith("num_batches_tracked"))
    YOLOv8Seg().load_state_dict(sd, strict=True)


def test_loader_refuses_foreign_globals(tmp_path):
    from sam6d_b200.fast_sam import load_fastsam_checkpoint
    path = str(tmp_path / "evil.pt")
    _fake_ultralytics_checkpoint(path, extra={"hook": os.getcwd})
    with pytest.raises(Exception, match="outside the allowlist"):
        load_fastsam_checkpoint(path)


def test_loader_lists_mismatching_keys(tmp_path):
    from sam6d_b200.fast_sam import load_fastsam_checkpoint
    path = str(tmp_path / "wrong.pt")
    torch.save({"model": nn.Sequential(nn.Conv2d(3, 4, 1)), "ema": None}, path)
    with pytest.raises(ValueError, match="missing .*model.0.bn.weight.*unexpected.*mis-shaped"):
        load_fastsam_checkpoint(path)


# ---------------------------------------------------------------------------------------------------------------- geometry
@pytest.mark.parametrize("hw,lb_shape,pad", [((480, 640), (480, 640), (0, 0)), ((720, 1280), (384, 640), (12, 0)), ((375, 500), (480, 640), (0, 0))])
def test_letterbox_and_scale_boxes(hw, lb_shape, pad):
    from oracle import fastsam_oracle as fo
    from sam6d_b200 import fast_sam, synth
    img = synth.make_fastsam_frame(*hw, seed=2)
    lb, (top, left) = fast_sam.letterbox(img)
    ref, _, _ = fo.letterbox(img)
    assert lb.shape[:2] == lb_shape and (top, left) == pad and np.array_equal(lb, ref)
    if top:
        assert (lb[:top] == 114).all() and (lb[-top:] == 114).all()
    boxes = torch.tensor([[10.0, 5.0, 300.5, 200.25], [-4.0, 20.0, 700.0, 500.0], [600.0, 370.0, 640.0, 384.0]])
    got = fast_sam.scale_boxes(lb_shape, boxes.clone(), hw)
    want = fo.scale_boxes(lb_shape, boxes.clone(), hw)
    assert torch.equal(got, want)
    gain = min(lb_shape[0] / hw[0], lb_shape[1] / hw[1])
    exp = ((boxes - torch.tensor([pad[1], pad[0], pad[1], pad[0]])) / gain)
    exp[:, [0, 2]] = exp[:, [0, 2]].clamp(0, hw[1])
    exp[:, [1, 3]] = exp[:, [1, 3]].clamp(0, hw[0])
    assert torch.allclose(got, exp)


def test_cascaded_max_pools_equal_wider_pools():
    """SPPF's three cascaded MaxPool2d(5, 1, 2) with -inf padding equal 5x5, 9x9 and 13x13 pools exactly (sam6d_yolo_sppf
    computes the latter directly): a window of a window, clipped at the border, is the wider window clipped at the border"""
    x = torch.randn(2, 7, 15, 20)
    y1 = F.max_pool2d(x, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    y3 = F.max_pool2d(y2, 5, 1, 2)
    assert torch.equal(y2, F.max_pool2d(x, 9, 1, 4)) and torch.equal(y3, F.max_pool2d(x, 13, 1, 6))


def test_cli_accepts_fastsam():
    from sam6d_b200.cli import ism_run_inference_custom as cli
    assert cli.get_parser().parse_args(["--segmentor_model", "fastsam"]).segmentor_model == "fastsam"
    with pytest.raises(ValueError):
        cli.main(["--segmentor_model", "yolo"])
