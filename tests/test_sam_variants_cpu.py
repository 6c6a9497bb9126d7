"""CPU: the three SAM backbones (vit_h, vit_l, vit_b) as the reference builds them.  sam_model_registry[t]() must have exactly the
state_dict layout of the vendored reference's sam_model_registry[t]() (tests/golden/sam_keys.pt, tools/make_golden.py sam_keys),
so that the released checkpoints load strictly; load_sam resolves the reference's checkpoint file names; the ISM CLI selects the
backbone with --sam_model_type."""
import os
from functools import partial

import pytest
import torch

TYPES = ("vit_h", "vit_l", "vit_b")
REF_FILES = {"vit_h": "sam_vit_h_4b8939.pth", "vit_l": "sam_vit_l_0b3195.pth", "vit_b": "sam_vit_b_01ec64.pth"}


@pytest.fixture(scope="module")
def keys_gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "sam_keys.pt"), weights_only=False)["types"]


def _synth_sam_state_dict(t):
    from sam6d_b200 import synth
    from sam6d_b200.sam import VIT_CONFIGS
    sd = {"image_encoder." + k: v for k, v in synth.make_sam_state_dict(**VIT_CONFIGS[t], seed=1).items()}
    sd.update(synth.make_sam_decoder_state_dict(seed=1))
    return sd


@pytest.mark.parametrize("t", TYPES)
def test_registry_matches_reference_layout(keys_gold, t):
    from sam6d_b200.sam_amg import sam_model_registry
    sam = sam_model_registry[t]()
    sd = sam.state_dict()
    gold = keys_gold[t]
    assert sorted((k, tuple(v.shape)) for k, v in sd.items()) == sorted(gold["keys"])
    assert sum(p.numel() for p in sam.parameters()) == gold["n_params"]
    with torch.no_grad():
        sam.load_state_dict(_synth_sam_state_dict(t), strict=True)


def test_registry_default_is_vit_h():
    from sam6d_b200.sam_amg import build_sam_vit_h, sam_model_registry
    assert sam_model_registry["default"] is build_sam_vit_h is sam_model_registry["vit_h"]
    assert set(sam_model_registry) == {"default", "vit_h", "vit_l", "vit_b"}


def test_vit_configs_match_oracle():
    from oracle import sam_oracle as so
    from sam6d_b200.sam import VIT_CONFIGS
    for t in TYPES:
        assert VIT_CONFIGS[t] == so.vit_cfg(t)


@pytest.mark.parametrize("embed_dim,num_heads", [(768, 8), (1280, 10), (1000, 16)])
def test_unsupported_head_dim_raises(embed_dim, num_heads):
    from sam6d_b200.sam import ImageEncoderViT
    with pytest.raises(ValueError, match=r"head dims \(64, 80\)"):
        ImageEncoderViT(depth=1, embed_dim=embed_dim, num_heads=num_heads, use_rel_pos=True, window_size=14,
                        norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def test_build_image_encoder_names():
    from sam6d_b200.sam import build_image_encoder
    enc = build_image_encoder("vit_b", precision="fp32")
    assert (enc.embed_dim, enc.num_heads, len(enc.blocks)) == (768, 12, 12)
    assert [i for i, b in enumerate(enc.blocks) if b.window_size == 0] == [2, 5, 8, 11]
    assert enc.blocks[2].attn.rel_pos_h.shape == (127, 64) and enc.blocks[0].attn.rel_pos_h.shape == (27, 64)
    with pytest.raises(ValueError, match="vit_x"):
        build_image_encoder("vit_x")


@pytest.mark.parametrize("t", TYPES)
def test_load_sam_names_missing_checkpoint(tmp_path, t):
    from sam6d_b200.sam_amg import load_sam, pretrained_weight_dict
    assert pretrained_weight_dict[t] == REF_FILES[t]
    with pytest.raises(FileNotFoundError, match=REF_FILES[t]):
        load_sam(t, str(tmp_path))


def test_load_sam_unknown_type(tmp_path):
    from sam6d_b200.sam_amg import load_sam
    with pytest.raises(ValueError, match="vit_q"):
        load_sam("vit_q", str(tmp_path))


def test_load_sam_reads_checkpoint_strictly(tmp_path):
    """a vit_b checkpoint under the reference's file name loads; a wrong backbone's checkpoint is refused"""
    from sam6d_b200.sam_amg import load_sam
    sd = _synth_sam_state_dict("vit_b")
    torch.save(sd, os.path.join(tmp_path, REF_FILES["vit_b"]))
    sam = load_sam("vit_b", str(tmp_path), precision="fp32")
    assert sam.image_encoder.precision == "fp32" and sam.image_encoder.embed_dim == 768
    got = sam.state_dict()
    for k in ("image_encoder.blocks.11.attn.rel_pos_w", "image_encoder.neck.2.weight", "mask_decoder.iou_token.weight"):
        assert torch.equal(got[k], sd[k])
    os.rename(os.path.join(tmp_path, REF_FILES["vit_b"]), os.path.join(tmp_path, REF_FILES["vit_l"]))
    with pytest.raises(RuntimeError, match="size mismatch|Missing key|Unexpected key"):
        load_sam("vit_l", str(tmp_path))


def test_cli_sam_model_type_flag():
    from sam6d_b200.cli import ism_run_inference_custom as cli
    ap = cli.get_parser()
    assert ap.parse_args([]).sam_model_type == "vit_h"
    for t in TYPES:
        assert ap.parse_args(["--sam_model_type", t]).sam_model_type == t
    with pytest.raises(SystemExit):
        ap.parse_args(["--sam_model_type", "vit_g"])
