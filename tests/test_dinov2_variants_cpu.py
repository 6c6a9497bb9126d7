"""CPU: the DINOv2 ViT-S/14, ViT-B/14 and ViT-g/14 descriptor backbones (sam6d_b200/dinov2.py, oracle/dinov2_variants_oracle.py)
against tests/golden/dinov2_variants.pt -- outputs and state_dict layouts of the reference's own vit_small / vit_base /
vit_giant2(ffn_layer="swiglufused") on seeded weights and the synthetic 6-proposal frame (tools/make_golden_dinov2_variants.py)."""
import os

import pytest
import torch

from oracle import dinov2_oracle as do, dinov2_variants_oracle as dvo

MODELS = ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitg14")


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "dinov2_variants.pt"), weights_only=False)


@pytest.mark.parametrize("name", MODELS)
def test_oracle_reproduces_fixture(gold, name):
    """full-depth fp32 forward of the oracle on the fixture's frame (the fixture was written where it equalled the reference
    bit for bit; another thread count may reorder the CPU GEMM sums, hence the 1e-5 bound)"""
    g = gold["models"][name]
    image, masks, boxes = do.make_proposals(P=gold["meta"]["P"], seed=gold["meta"]["seed"])
    assert torch.equal(boxes, gold["boxes"]) and image.double().sum().item() == gold["input_checksum"]["image"]
    sd = dvo.make_state_dict(name, seed=gold["meta"]["seed"])
    assert {k: tuple(v.shape) for k, v in sd.items()} == g["state_dict_shapes"]
    with torch.no_grad():
        rgbs = do.process_rgb_proposals(image, masks.clone(), boxes)
        pm = do.process_masks_proposals(masks.clone(), boxes)
        cls, pf, keep = dvo.cls_and_patch_features(sd, rgbs, pm, name)
    assert torch.equal(keep, g["keep"])
    torch.testing.assert_close(cls, g["cls"], atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(pf[:, ::gold["meta"]["patch_step"], ::gold["meta"]["channel_step"]], g["patch_sub"], atol=1e-5, rtol=0)


@pytest.mark.parametrize("name", MODELS)
def test_state_dict_layout_matches_reference(gold, name):
    from sam6d_b200.dinov2 import CustomDINOv2, descriptor_size
    with torch.device("meta"):
        d = CustomDINOv2(name)
    g = gold["models"][name]
    assert {k: tuple(v.shape) for k, v in d.model.state_dict().items()} == g["state_dict_shapes"]
    assert sum(p.numel() for p in d.model.parameters()) == g["num_params"]
    assert d.model.embed_dim == descriptor_size[name] == g["arch"]["embed_dim"]
    assert (d.model.depth, d.model.num_heads, d.model.ffn_layer) == (g["arch"]["depth"], g["arch"]["num_heads"], g["arch"]["ffn_layer"])


def test_model_names():
    from sam6d_b200 import dinov2 as sd
    assert set(sd.descriptor_map) == set(sd.descriptor_size) == set(dvo.ARCHS)
    with torch.device("meta"):
        for name, (C, heads, depth, ffn) in dvo.ARCHS.items():
            m = sd.CustomDINOv2(name).model
            assert (m.embed_dim, m.num_heads, m.depth, m.ffn_layer) == (C, heads, depth, ffn)
        assert sd.CustomDINOv2().model.ffn_layer == "mlp" and sd.CustomDINOv2().model_name == "dinov2_vitl14"
        for bad in ("dinov2_vits14_reg", "dinov2_vitg14_reg", "dinov2_vith14"):
            with pytest.raises(NotImplementedError):
                sd.CustomDINOv2(bad)
        with pytest.raises(NotImplementedError):
            sd.vit_large(ffn_layer="swiglu")
        # the reference builds ViT-g with an Mlp when asked to; that configuration stays constructible
        assert "blocks.0.mlp.fc1.weight" in sd.vit_giant2().state_dict()


def test_swiglu_row_packing():
    """gate rows [128t, +128) then up rows [128t, +128): the layout gemm_tma(act=3) reads one 256-row N tile of"""
    from sam6d_b200.ops import pack_swiglu_rows
    H = 384
    w = torch.arange(2 * H, dtype=torch.float32)[:, None].expand(2 * H, 3).contiguous()
    p = pack_swiglu_rows(w)
    for t in range(H // 128):
        assert torch.equal(p[256 * t:256 * t + 128, 0], torch.arange(128 * t, 128 * t + 128, dtype=torch.float32))
        assert torch.equal(p[256 * t + 128:256 * t + 256, 0], torch.arange(H + 128 * t, H + 128 * t + 128, dtype=torch.float32))
    assert torch.equal(pack_swiglu_rows(w[:, 0]), p[:, 0])
    with pytest.raises(ValueError):
        pack_swiglu_rows(torch.zeros(2 * 100, 4))


def test_default_state_dict_draw_unchanged(gold):
    """make_state_dict(seed=1) without an architecture still draws the ViT-L/14 tensors tests/golden/dinov2.pt was made from"""
    sd = do.make_state_dict(seed=1)
    assert {k: v.double().sum().item() for k, v in sd.items()} == gold["meta"]["default_draw_checksum"]
    assert torch.equal(dvo.make_state_dict("dinov2_vitl14", seed=1)["blocks.0.mlp.fc2.bias"], sd["blocks.0.mlp.fc2.bias"])


def test_cli_flag():
    from sam6d_b200.cli import ism_run_inference_custom as cli
    ap = cli.get_parser()
    assert ap.parse_args([]).dinov2_model == "dinov2_vitl14"
    for name in ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14"):
        args = ap.parse_args(["--dinov2_model", name, "--checkpoint_dir", "/ck"])
        assert cli._dino_checkpoint(args) == os.path.join("/ck", "dinov2", f"{name}_pretrain.pth")
    with pytest.raises(SystemExit):
        ap.parse_args(["--dinov2_model", "dinov2_vitl14_reg"])
