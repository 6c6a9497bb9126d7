"""tools/make_golden_vit_gather.py -- writes tests/golden/vit_pixel_feats.json: the reference's own get_chosen_pixel_feats
(Pose_Estimation_Model/utils/model_utils.py, imported unmodified) on a seeded feature map and pixel choice.

Usage: python tools/make_golden_vit_gather.py <SAM-6D/Pose_Estimation_Model directory of the reference> [out.json]"""
import builtins
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    pem = sys.argv[1]
    builtins.__POINTNET2_SETUP__ = True            # model_utils imports pointnet2; its compiled extension is not needed here
    sys.path[:0] = [os.path.join(pem, "utils"), os.path.join(pem, "model", "pointnet2")]
    import model_utils as mu
    g = torch.Generator().manual_seed(0)
    img = torch.randn(2, 2, 5, 6, generator=g)
    choose = torch.randint(0, 5 * 6, (2, 12), generator=g)
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "tests", "golden", "vit_pixel_feats.json")
    with open(out, "w") as fh:
        json.dump({"img": img.tolist(), "choose": choose.tolist(), "feats": mu.get_chosen_pixel_feats(img, choose).tolist()}, fh)
    print(f"wrote {out}")


if __name__ == "__main__":
    main()
