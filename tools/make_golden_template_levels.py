"""tools/make_golden_template_levels.py -- DEV CONTAINER ONLY (needs the reference checkout).

Copies the reference's CNOS level-1 and level-2 template poses (ISM/utils/poses/predefined_poses/{cam,obj}_poses_level{1,2}.npy,
written by ISM/utils/poses/create_template_poses.py in Blender) and the indices of the level-0 / level-1 views among the
level-2 ones (idx_all_level{0,1}_in_level2.npy, read by load_index_level_in_level2) into tests/golden/template_poses_levels.pt,
so tests/test_template_levels_cpu.py can pin sam6d_b200.render.template_poses() against them without the reference.
The level-0 files are tests/golden/template_poses_level0.pt (tools/make_golden_render.py).

Usage: python tools/make_golden_template_levels.py"""
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = "/root/reference/SAM-6D/Instance_Segmentation_Model/utils/poses/predefined_poses"


def main():
    out = {}
    for level in (1, 2):
        for k in ("cam_poses", "obj_poses"):
            out[f"{k}_level{level}"] = torch.from_numpy(np.load(os.path.join(SRC, f"{k}_level{level}.npy")).astype(np.float64))
    for level in (0, 1):
        out[f"idx_all_level{level}_in_level2"] = torch.from_numpy(np.load(os.path.join(SRC, f"idx_all_level{level}_in_level2.npy")).astype(np.int64))
    path = os.path.join(ROOT, "tests", "golden", "template_poses_levels.pt")
    torch.save(out, path)
    print("wrote", path, {k: tuple(v.shape) for k, v in out.items()})


if __name__ == "__main__":
    main()
