"""tools/make_golden_sam_predictor.py -- DEV CONTAINER ONLY (needs /root/reference).

Pins oracle/sam_predictor_oracle.py against the vendored reference modules (ISM/segment_anything: PromptEncoder, MaskDecoder,
TwoWayTransformer, Sam, SamPredictor, ResizeLongestSide) on seeded weights and a synthetic image embedding, and writes
tests/golden/sam_predictor.pt.  The predictor wraps a stand-in image encoder (img_size 1024) and gets the embedding injected
as `features`: the encoders have fixtures of their own.

Usage: python tools/make_golden_sam_predictor.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference/SAM-6D/Instance_Segmentation_Model")

from oracle import sam_dec_oracle as so  # noqa: E402
from oracle import sam_predictor_oracle as sp  # noqa: E402
from sam6d_b200 import synth  # noqa: E402

SIZES = ((480, 640), (640, 480))


def _reference_predictor(sd, feat, original_size):
    from segment_anything.modeling import MaskDecoder, PromptEncoder, Sam, TwoWayTransformer
    from segment_anything.predictor import SamPredictor
    pe = PromptEncoder(embed_dim=256, image_embedding_size=(64, 64), input_image_size=(1024, 1024), mask_in_chans=16)
    md = MaskDecoder(num_multimask_outputs=3, transformer=TwoWayTransformer(depth=2, embedding_dim=256, mlp_dim=2048, num_heads=8),
                     transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256)
    enc = torch.nn.Module()
    enc.img_size = 1024
    sam = Sam(enc, pe, md).eval()
    sam.prompt_encoder.load_state_dict({k[len("prompt_encoder."):]: v for k, v in sd.items() if k.startswith("prompt_encoder.")}, strict=True)
    sam.mask_decoder.load_state_dict({k[len("mask_decoder."):]: v for k, v in sd.items() if k.startswith("mask_decoder.")}, strict=True)
    p = SamPredictor(sam)
    p.features = feat
    p.original_size = original_size
    p.input_size = p.transform.get_preprocess_shape(original_size[0], original_size[1], 1024)
    p.is_image_set = True
    return p


def main():
    torch.set_num_threads(8)
    sd = so.make_state_dict(seed=1)
    feat = synth.make_image_embedding(seed=1)
    gold = dict(meta=dict(source="segment_anything SamPredictor / PromptEncoder / MaskDecoder / Sam / ResizeLongestSide imported from "
                                 "/root/reference", torch=torch.__version__, seed=1, sizes=SIZES),
                feat_checksum=feat.double().sum().item(), sizes={})
    for size in SIZES:
        ref = _reference_predictor(sd, feat, size)
        mine = sp.run_cases(sd, feat, size)
        rec, outs = {}, {}
        for name, c in sp.make_cases(size).items():
            kw = sp.resolve_kwargs(name, c["kwargs"], outs.get("click"))
            with torch.no_grad():
                if c["api"] == "predict_torch":
                    b = ref.transform.apply_boxes_torch(torch.as_tensor(kw["boxes"], dtype=torch.float), size)
                    assert torch.equal(b, sp.apply_boxes_torch(torch.as_tensor(kw["boxes"], dtype=torch.float), size))
                    r = ref.predict_torch(None, None, boxes=b, multimask_output=kw["multimask_output"])
                else:
                    r = tuple(torch.as_tensor(a) for a in ref.predict(**kw))
            outs[name] = r
            masks, iou, low = r
            for what, a, b in (("masks", masks, mine[name][0]), ("iou", iou, mine[name][1]), ("low-res", low, mine[name][2])):
                assert a.shape == b.shape, (name, what, a.shape, b.shape)
                d = (a.double() - b.double()).abs().max().item()
                assert d == 0.0, (size, name, what, d)
            full = masks if masks.dtype != torch.bool else None
            rec[name] = dict(low_sub=low[..., ::8, ::8].clone(), low_abs_mean=low.abs().mean().item(), iou=iou.clone(),
                             mask_area=(masks > 0 if full is not None else masks).flatten(-2).sum(-1).clone(),
                             full_sub=masks[..., ::16, ::16].clone(), shape=tuple(masks.shape))
            print(f"  {size} {name:16s} masks {tuple(masks.shape)} iou {[round(v, 4) for v in iou.flatten().tolist()[:4]]} "
                  f"max|ref - oracle| = 0")
        # ResizeLongestSide: the numpy and torch coordinate / box transforms
        c = sp.make_cases(size)
        pts = c["clicks26"]["kwargs"]["point_coords"]
        bxs = c["boxes16_torch"]["kwargs"]["boxes"]
        rec["transform"] = dict(points=torch.as_tensor(pts), boxes=torch.as_tensor(bxs),
                                coords=torch.as_tensor(ref.transform.apply_coords(pts, size)),
                                boxes_t=torch.as_tensor(ref.transform.apply_boxes(bxs, size)),
                                coords_torch=ref.transform.apply_coords_torch(torch.as_tensor(pts, dtype=torch.float), size),
                                boxes_torch=ref.transform.apply_boxes_torch(torch.as_tensor(bxs, dtype=torch.float), size),
                                preprocess_shape=ref.transform.get_preprocess_shape(size[0], size[1], 1024))
        assert np.array_equal(rec["transform"]["coords"].numpy(), sp.apply_coords(pts, size))
        gold["sizes"][size] = rec
    path = os.path.join(ROOT, "tests", "golden", "sam_predictor.pt")
    torch.save(gold, path)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
