"""tools/make_golden_dinov2_variants.py -- DEV CONTAINER ONLY (needs /root/reference).

Pins oracle/dinov2_variants_oracle.py against the reference's OWN modules, imported unmodified from /root/reference:
    ISM/model/vision_transformer.py  vit_small / vit_base / vit_giant2(patch_size=14, img_size=518, init_values=1.0, block_chunks=0,
                                     ffn_layer="mlp" / "mlp" / "swiglufused")   (= dinov2_vits14 / vitb14 / vitg14)
    ISM/model/dinov2.py              CustomDINOv2.process_rgb_proposals / process_masks_proposals / compute_cls_and_patch_features
    ISM/model/loss.py                MaskedPatch_MatrixSimilarity.compute_straight / compute_visible_ratio
and writes tests/golden/dinov2_variants.pt: per backbone the content of tests/golden/dinov2.pt (cls tokens, masked patch tokens
subsampled in tokens and channels, validity pattern, appearance score / visible ratio) on the same seeded 6-proposal frame, full depth, plus the
state_dict key names and shapes of the reference module.  Weights and the frame are regenerated from their seeds, never stored.

ViT-g is built with ffn_layer="swiglufused": the reference's CustomDINOv2 passes the default "mlp", which cannot load the published
SwiGLU checkpoint (INTEGRATION.md section 3c).  Without xformers, SwiGLUFFNFused is the reference's own SwiGLUFFN.

Usage: python tools/make_golden_dinov2_variants.py   (a few minutes on the CPU: ViT-g is ~3.6 TFLOP per pass)"""
import os
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import dinov2_oracle as do, dinov2_variants_oracle as dvo, ism_oracle as io  # noqa: E402
from ref_ism_import import import_reference_ism, STUBBED  # noqa: E402

MODELS = ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitg14")
PATCH_STEP = 7           # masked patch tokens kept in the fixture: every 7th of the 256 (varied grid rows and columns) ...
CHANNEL_STEP = 12        # ... and every 12th channel: keeps the fixture small (the cls tokens are stored whole)


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    loss, _ = import_reference_ism()
    from model import vision_transformer as vits, dinov2 as rdino           # the reference's modules
    from utils.bbox_utils import CropResizePad
    import torchvision.transforms as T
    print("stubbed third-party imports:", STUBBED)
    image, masks, boxes = do.make_proposals(P=6, seed=1)
    gold = dict(meta=dict(source="ISM/model/vision_transformer.py vit_small / vit_base / vit_giant2 + ISM/model/dinov2.py + ISM/utils/bbox_utils.py "
                                 "+ ISM/model/loss.py imported from /root/reference (CPU, fp32)", torch=torch.__version__, seed=1, P=6,
                          patch_step=PATCH_STEP, channel_step=CHANNEL_STEP, stubbed_imports=list(STUBBED)),
                boxes=boxes, input_checksum=dict(image=image.double().sum().item(), masks=masks.double().sum().item()), models={})
    # make_state_dict(seed=1) without an architecture must keep drawing the ViT-L/14 tensors tests/golden/dinov2.pt was made from
    gold["meta"]["default_draw_checksum"] = {k: v.double().sum().item() for k, v in do.make_state_dict(seed=1).items()}
    D = rdino.CustomDINOv2
    for name in MODELS:
        C, heads, depth, ffn = dvo.ARCHS[name]
        assert rdino.descriptor_size[name] == C
        t0 = time.time()
        sd = dvo.make_state_dict(name, seed=1)
        ref = getattr(vits, rdino.descriptor_map[name])(patch_size=14, img_size=518, init_values=1.0, ffn_layer=ffn, block_chunks=0,
                                                         num_register_tokens=0, interpolate_antialias=False, interpolate_offset=0.1).eval()
        keys = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
        print(f"{name}: reference {rdino.descriptor_map[name]} accepted the oracle state_dict (strict):", ref.load_state_dict(sd, strict=True))
        host = types.SimpleNamespace(model=ref, rgb_normalize=T.Compose([T.ToTensor(), T.Normalize(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))]),
                                     rgb_proposal_processor=CropResizePad(224), patch_kernel=torch.nn.AvgPool2d(kernel_size=14, stride=14),
                                     validpatch_thresh=0.5, chunk_size=16)
        with torch.no_grad():
            r_rgbs = D.process_rgb_proposals(host, image.numpy(), masks.clone(), boxes)
            r_masks = D.process_masks_proposals(host, masks.clone(), boxes)
            r_cls, r_patch = D.compute_cls_and_patch_features(host, r_rgbs, r_masks)
            o_rgbs = do.process_rgb_proposals(image, masks.clone(), boxes)
            o_masks = do.process_masks_proposals(masks.clone(), boxes)
            o_cls, o_patch, o_keep = dvo.cls_and_patch_features(sd, o_rgbs, o_masks, name)
        for what, a, b in (("cls tokens", r_cls, o_cls), ("masked patch tokens", r_patch, o_patch)):
            d = (a - b).abs().max().item()
            print(f"  {what:22s} max|ref - oracle| = {d:.3e}")
            assert d == 0.0, (name, what)
        m = loss.MaskedPatch_MatrixSimilarity(metric="cosine", chunk_size=64)
        ref_patch = r_patch.roll(1, dims=0)
        r_appe, r_vis = m.compute_straight(r_patch, ref_patch), m.compute_visible_ratio(r_patch, ref_patch, 0.5)
        assert torch.equal(io.appearance_score(o_patch, o_patch.roll(1, dims=0)), r_appe)
        assert torch.equal(io.visible_ratio(o_patch, o_patch.roll(1, dims=0), 0.5), r_vis)
        gold["models"][name] = dict(arch=dict(embed_dim=C, num_heads=heads, depth=depth, ffn_layer=ffn), state_dict_shapes=keys,
                                    num_params=sum(p.numel() for p in ref.parameters()), cls=r_cls.clone(),
                                    patch_sub=r_patch[:, ::PATCH_STEP, ::CHANNEL_STEP].clone(), keep=o_keep, appe=r_appe, vis=r_vis)
        print(f"  {len(keys)} state_dict entries, {gold['models'][name]['num_params']} parameters, {time.time() - t0:.0f} s")
        del ref, sd
    path = os.path.join(ROOT, "tests", "golden", "dinov2_variants.pt")
    torch.save(gold, path)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
