"""tools/make_golden_render.py -- DEV CONTAINER ONLY (needs /root/reference).

Copies the reference's CNOS level-0 template poses (ISM/utils/poses/predefined_poses/{cam,obj}_poses_level0.npy, written by
ISM/utils/poses/create_template_poses.py in Blender) into tests/golden/template_poses_level0.pt as float64 tensors, so
tests/test_render_cpu.py can pin sam6d_b200.render.level0_template_poses() against them without the reference.

Usage: python tools/make_golden_render.py"""
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = "/root/reference/SAM-6D/Instance_Segmentation_Model/utils/poses/predefined_poses"


def main():
    out = {k: torch.from_numpy(np.load(os.path.join(SRC, f"{k}_level0.npy")).astype(np.float64)) for k in ("cam_poses", "obj_poses")}
    path = os.path.join(ROOT, "tests", "golden", "template_poses_level0.pt")
    torch.save(out, path)
    print("wrote", path, {k: tuple(v.shape) for k, v in out.items()})


if __name__ == "__main__":
    main()
