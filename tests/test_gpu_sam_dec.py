"""GPU: SAM prompt encoder / mask decoder / automatic-mask-generator post-processing (SURVEY.md 8f row N4: sam6d_b200/sam_amg.py,
csrc/sam_dec.cu) against tests/golden/sam_dec.pt -- outputs of the vendored reference modules (PromptEncoder, MaskDecoder,
TwoWayTransformer, Sam.postprocess_masks, utils.amg) on seeded weights and a synthetic image embedding
(tools/make_golden_sam_dec.py) -- and against the pinned oracle for inputs the fixture does not hold."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import sam_dec_oracle as so      # noqa: E402
from sam6d_b200 import synth                 # noqa: E402


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "sam_dec.pt"), weights_only=False)


@pytest.fixture(scope="module")
def amg(gold):
    """decoder + generator with the seeded weights; the image embedding is injected (the ViT-H encoder has its own tests)"""
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator, MaskDecoder, PromptEncoder, Sam
    sd = so.make_state_dict(seed=gold["meta"]["seed"])
    enc = torch.nn.Module()
    enc.img_size = 1024
    sam = Sam(enc, PromptEncoder(), MaskDecoder()).cuda().eval()
    sam.prompt_encoder.load_state_dict({k[len("prompt_encoder."):]: v for k, v in sd.items() if k.startswith("prompt_encoder.")}, strict=True)
    sam.mask_decoder.load_state_dict({k[len("mask_decoder."):]: v for k, v in sd.items() if k.startswith("mask_decoder.")}, strict=True)
    g = CustomSamAutomaticMaskGenerator(sam, stability_score_thresh=0.95, points_per_side=8)
    feat = synth.make_image_embedding(seed=gold["meta"]["seed"])
    assert feat.double().sum().item() == gold["feat_checksum"]
    g.features = feat.cuda()
    g.image_pe_rows = sam.prompt_encoder.dense_pe_rows()
    g.original_size, g.input_size = (480, 640), so.preprocess_shape(480, 640)
    return g


def test_prompt_encoder(gold, amg):
    pe = amg.sam.prompt_encoder
    torch.testing.assert_close(pe.get_dense_pe().cpu()[:, :, ::8, ::8], gold["dense_pe_sub"], atol=2e-5, rtol=0)
    pts = so.build_point_grid(8) * np.array([640, 480])[None, :]
    c = torch.as_tensor(so.apply_coords(pts, (480, 640))).cuda()[:, None, :]
    sparse, dense = pe(points=(c, torch.ones(64, 1, dtype=torch.int, device="cuda")))
    torch.testing.assert_close(sparse.cpu(), gold["sparse"], atol=3e-5, rtol=0)
    assert dense.shape == (64, 256, 64, 64)


def test_mask_decoder_matches_reference(gold, amg):
    """64 point prompts through the two-way transformer and the upscaling head: low-res mask logits and IoU predictions against
    the reference decoder (fp32 on the CPU).  Image-side operands are bf16 on the tensor cores: bounds = measured drift + margin."""
    pts = so.build_point_grid(8) * np.array([640, 480])[None, :]
    _, _, _, low, iou, _ = amg.process_batch(pts)
    low = low.view(64, 3, 256, 256).cpu()
    ref = gold["low_sub"]
    err = (low[:, :, ::8, ::8] - ref).abs()
    rel = (err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    sign = ((low[:, :, ::8, ::8] > 0) == (ref > 0)).float().mean().item()
    ierr = (iou.cpu() - gold["iou_all"]).abs().max().item()
    print(f"mask decoder: rel rms error of the low-res logits {rel:.3e} (|ref| mean {gold['low_abs_mean']:.1f}), sign agreement {sign:.5f}, "
          f"max |iou - ref| {ierr:.3e}")
    assert rel < 3e-2 and sign > 0.99 and ierr < 2e-2


def test_postprocess_stats_and_binarize_against_oracle(amg):
    """Sam.postprocess_masks + stability counts + boxes + binarisation evaluated per output pixel, on smooth synthetic low-res
    logits, against the reference formulation (two F.interpolate calls, utils.amg helpers restated in the oracle)"""
    from sam6d_b200 import _lib
    g = torch.Generator().manual_seed(4)
    n = 12
    base = torch.nn.functional.interpolate(torch.randn(n, 1, 12, 12, generator=g) * 6, size=(256, 256), mode="bicubic")[:, 0]
    low = (base + 0.3 * torch.randn(n, 256, 256, generator=g)).contiguous()
    low[3] = -5.0                                                  # an empty mask
    ref = so.postprocess_masks(low[None], (768, 1024), (480, 640))[0]
    stats = torch.empty(n, 8, dtype=torch.int32, device="cuda")
    low_d = low.cuda()
    _lib.call("sam6d_sam_mask_stats", low_d, n, 256, 1024, 768, 1024, 480, 640, 0.0, 1.0, stats)
    s = stats.cpu()
    hi, lo = (ref > 1.0).flatten(1).sum(1), (ref > -1.0).flatten(1).sum(1)
    print("count(>1) gpu/ref", s[:, 0].tolist(), hi.tolist())
    assert (s[:, 0] - hi).abs().max() <= 3 and (s[:, 1] - lo).abs().max() <= 3         # borderline pixels: float op order
    boxes = so.batched_mask_to_box(ref > 0.0)
    mine = s[:, 2:6].long()
    mine[(mine[:, 2] < mine[:, 0]) | (mine[:, 3] < mine[:, 1])] = 0
    assert (mine - boxes).abs().max() <= 1
    sel = torch.arange(n, dtype=torch.int32, device="cuda")
    out = torch.empty(n, 480, 640, dtype=torch.uint8, device="cuda")
    _lib.call("sam6d_sam_mask_binarize", low_d, sel, n, 256, 1024, 768, 1024, 480, 640, 0.0, out)
    mism = (out.cpu().bool() != (ref > 0.0)).float().mean().item()
    assert mism < 2e-5, mism


def test_nms_matches_torchvision_semantics(amg):
    g = torch.Generator().manual_seed(0)
    for n in (1, 7, 300, 3000):
        xy = torch.randint(0, 400, (n, 2), generator=g).float()
        wh = torch.randint(20, 200, (n, 2), generator=g).float()
        b = torch.cat([xy, xy + wh], dim=1)
        sc = torch.rand(n, generator=g)
        assert torch.equal(amg.nms(b.cuda(), sc.cuda(), 0.7).cpu(), so.nms(b, sc, 0.7))
    assert amg.nms(torch.zeros(0, 4).cuda(), torch.zeros(0).cuda(), 0.7).numel() == 0


def test_process_batch_filters(gold, amg):
    """the kept set of one 64-prompt batch: predicted-IoU and stability filters are thresholds, so masks that sit on a threshold may
    flip under bf16; everything kept by both sides must agree in its box"""
    pts = so.build_point_grid(8) * np.array([640, 480])[None, :]
    masks, boxes, iou, low, iou_all, stats = amg.process_batch(pts)
    st = stats.cpu()
    stab = st[:, 0].float() / st[:, 1].float()
    print("stability gpu vs ref: max |diff|", (stab - gold["stability_all"]).abs().max().item())
    mine = set(torch.nonzero((iou_all.cpu() > 0.88) & (stab >= 0.95)).flatten().tolist())
    ref = set(gold["kept_index"].tolist())
    print(f"kept: gpu {len(mine)}, reference {len(ref)}, common {len(mine & ref)}")
    assert len(mine & ref) >= 0.8 * len(ref) and len(mine) <= 1.25 * len(ref)
    assert masks.shape == (len(mine), 480, 640) and boxes.shape == (len(mine), 4)
    area = masks.flatten(1).sum(1).cpu()
    ref_area = dict(zip(gold["kept_index"].tolist(), gold["mask_area"].tolist()))
    ref_box = dict(zip(gold["kept_index"].tolist(), gold["boxes"].tolist()))
    for j, idx in enumerate(sorted(mine)):
        if idx in ref:
            assert abs(int(area[j]) - ref_area[idx]) <= 0.01 * ref_area[idx] + 20
            assert max(abs(a - b) for a, b in zip(boxes[j].tolist(), ref_box[idx])) <= 2
