"""CPU: the SAM predictor's oracle (oracle/sam_predictor_oracle.py) against tests/golden/sam_predictor.pt -- outputs of the
vendored reference SamPredictor (tools/make_golden_sam_predictor.py) -- plus ResizeLongestSide and the input checks of
sam6d_b200.sam_amg that raise before any device work."""
import os

import numpy as np
import pytest
import torch

from oracle import sam_dec_oracle as so
from oracle import sam_predictor_oracle as sp
from sam6d_b200 import synth


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "sam_predictor.pt"), weights_only=False)


@pytest.mark.parametrize("size", [(480, 640), (640, 480)])
def test_oracle_matches_reference_predictor(gold, size):
    """every prompt case (clicks, labels -1 / 0 / 1, a box, box + clicks, a mask input, 16 boxes, 26 clicks, logits) bit for bit"""
    sd = so.make_state_dict(seed=gold["meta"]["seed"])
    feat = synth.make_image_embedding(seed=gold["meta"]["seed"])
    assert feat.double().sum().item() == gold["feat_checksum"]
    out = sp.run_cases(sd, feat, size)
    ref = gold["sizes"][size]
    assert set(out) == set(ref) - {"transform"}
    for name, (masks, iou, low) in out.items():
        r = ref[name]
        assert tuple(masks.shape) == r["shape"], name
        assert torch.equal(low[..., ::8, ::8], r["low_sub"]), name
        assert torch.equal(iou, r["iou"]), name
        assert torch.equal(masks[..., ::16, ::16], r["full_sub"]), name
        area = (masks > 0 if masks.dtype != torch.bool else masks).flatten(-2).sum(-1)
        assert torch.equal(area, r["mask_area"]), name


@pytest.mark.parametrize("size", [(480, 640), (640, 480)])
def test_resize_longest_side_matches_reference(gold, size):
    from sam6d_b200.sam_amg import ResizeLongestSide
    t = gold["sizes"][size]["transform"]
    tr = ResizeLongestSide(1024)
    pts, boxes = t["points"].numpy(), t["boxes"].numpy()
    assert tr.get_preprocess_shape(size[0], size[1], 1024) == t["preprocess_shape"]
    assert np.array_equal(tr.apply_coords(pts, size), t["coords"].numpy())
    assert np.array_equal(tr.apply_boxes(boxes, size), t["boxes_t"].numpy())
    assert torch.equal(tr.apply_coords_torch(torch.as_tensor(pts, dtype=torch.float), size), t["coords_torch"])
    assert torch.equal(tr.apply_boxes_torch(torch.as_tensor(boxes, dtype=torch.float), size), t["boxes_torch"])
    img = np.zeros(size + (3,), dtype=np.uint8)
    assert tr.apply_image(img).shape[:2] == t["preprocess_shape"]


def _cpu_sam():
    from sam6d_b200.sam_amg import MaskDecoder, PromptEncoder, Sam
    enc = torch.nn.Module()
    enc.img_size = 1024
    return Sam(enc, PromptEncoder(), MaskDecoder()).eval()


def test_prompt_checks_raise_before_any_launch():
    """on a CPU model: a kernel launch would fail with another error, so each ValueError shows the check ran first"""
    pe = _cpu_sam().prompt_encoder
    one = (torch.zeros(2, 1, 2), torch.ones(2, 1, dtype=torch.int))
    with pytest.raises(ValueError, match=r"\(B, 1, 256, 256\)"):
        pe(points=None, boxes=None, masks=torch.zeros(1, 256, 256))
    with pytest.raises(ValueError, match=r"\(B, 1, 256, 256\)"):
        pe(points=None, boxes=None, masks=torch.zeros(1, 1, 128, 128))
    with pytest.raises(ValueError, match="batch sizes differ"):
        pe(points=one, boxes=torch.zeros(3, 4), masks=None)
    with pytest.raises(ValueError, match="batch sizes differ"):
        pe(points=one, boxes=None, masks=torch.zeros(1, 1, 256, 256))
    with pytest.raises(ValueError, match="batch sizes differ"):
        pe(points=(torch.zeros(2, 3, 2), torch.ones(1, 3)), boxes=None, masks=None)
    with pytest.raises(ValueError, match="at most 27"):                      # 27 clicks + padding point
        pe(points=(torch.zeros(1, 27, 2), torch.ones(1, 27)), boxes=None, masks=None)
    with pytest.raises(ValueError, match="at most 27"):                      # 26 clicks + a box
        pe(points=(torch.zeros(1, 26, 2), torch.ones(1, 26)), boxes=torch.zeros(1, 4), masks=None)
    md = _cpu_sam().mask_decoder
    with pytest.raises(ValueError, match="at most 27"):
        md(torch.zeros(1, 256, 64, 64), torch.zeros(4096, 256), torch.zeros(1, 28, 256), torch.zeros(1, 256, 64, 64), True)


def test_predict_before_set_image_raises():
    from sam6d_b200.sam_amg import SamPredictor
    p = SamPredictor(_cpu_sam())
    assert not p.is_image_set and p.features is None and p.transform.target_length == 1024
    with pytest.raises(RuntimeError, match=r"An image must be set with \.set_image\(\.\.\.\) before mask prediction\."):
        p.predict(point_coords=np.array([[10.0, 10.0]]), point_labels=np.array([1]))
    with pytest.raises(RuntimeError, match=r"before mask prediction"):
        p.predict_torch(None, None, boxes=torch.zeros(1, 4))
    with pytest.raises(RuntimeError, match=r"to generate an embedding"):
        p.get_image_embedding()


def test_load_sam_predictor_missing_checkpoint(tmp_path):
    from sam6d_b200.sam_amg import load_sam_predictor
    with pytest.raises(FileNotFoundError, match="sam_vit_b_01ec64.pth"):
        load_sam_predictor("vit_b", str(tmp_path), "cpu")
    with pytest.raises(ValueError, match="unknown SAM model_type"):
        load_sam_predictor("vit_x", str(tmp_path), "cpu")
