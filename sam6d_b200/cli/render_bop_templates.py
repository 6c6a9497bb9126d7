"""Drop-in for SAM-6D/Render/render_bop_templates.py: the 42 template views of every object of a BOP dataset, rendered on the
GPU several objects per rasteriser call (sam6d_b200/render.py) instead of one BlenderProc scene per view.

    python -m sam6d_b200.cli.render_bop_templates --dataset_name ycbv [--bop_root Data/BOP --output_dir Data/BOP-Templates]

Reads <bop_root>/<dataset>/models/models_info.json (models_cad for T-LESS) and obj_XXXXXX.ply, and writes
<output_dir>/<dataset>/obj_XXXXXX/{rgb_i.png, mask_i.png, xyz_i.npy (mm, float16), template_poses.npy (translation in m)}.
Framing as in the reference: scale 1/diameter at distance 2, i.e. d = 2 x diameter in model units.  T-LESS is painted in a
uniform 0.4 grey; other models use their texture, else vertex colours, else grey 0.8.  Views (including
--level_templates / --pose_distribution and the directory layout they give) and shading: see render_custom_templates."""
import argparse
import json
import os

import numpy as np

from .. import meshio, render
from .render_custom_templates import BLENDER_DEFAULT_GREY, render_views, to_metres, view_set, view_set_parser, write_views

OBJECTS_PER_CALL = 8          # bounds the device outputs of one call: 8 x 42 views x 512^2 x 18 B = 1.6 GB (fewer objects with more views)


def get_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dataset_name', help="The name of bop datasets")
    # not in the reference (it hard-codes ../Data/BOP and ../Data/BOP-Templates next to its own folder)
    ap.add_argument('--bop_root', default=os.path.join("Data", "BOP"), help="folder holding <dataset_name>/models")
    ap.add_argument('--output_dir', default=os.path.join("Data", "BOP-Templates"), help="templates go to <output_dir>/<dataset_name>/obj_XXXXXX")
    ap.add_argument('--size', type=int, default=512, help="template width and height in pixels (the reference renders 512)")
    ap.add_argument('--poses', default=None, help="(T,4,4) .npy of object -> camera poses, translation in mm at 1000 mm "
                                                  "(the reference's obj_poses_level0.npy); default: level0_template_poses()")
    return ap


def parse_args(argv=None):
    """get_parser()'s arguments plus render_custom_templates.view_set_parser()'s, in one namespace"""
    args, rest = get_parser().parse_known_args(argv)
    view_set_parser().parse_args(rest, namespace=args)
    return args


def main(argv=None):
    args = parse_args(argv)
    per_call = max(1, OBJECTS_PER_CALL * render.VIEW_COUNTS[0] // len(view_set(1.0, args.poses, args.level_templates, args.pose_distribution)[0]))
    tless = args.dataset_name == 'tless'
    model_path = os.path.join(args.bop_root, args.dataset_name, 'models_cad' if tless else 'models')
    models_info = json.load(open(os.path.join(model_path, 'models_info.json')))
    obj_ids = list(models_info.keys())
    for c0 in range(0, len(obj_ids), per_call):
        ids = obj_ids[c0:c0 + per_call]
        meshes, poses, greys = [], [], []
        for obj_id in ids:
            mesh = meshio.load_ply_mesh(os.path.join(model_path, f'obj_{int(obj_id):06d}.ply'))
            if tless:
                mesh.colors = mesh.uv = mesh.texture = None
            meshes.append(render.upload(mesh))
            poses.append(view_set(2.0 * float(models_info[obj_id]['diameter']), args.poses, args.level_templates, args.pose_distribution)[0])
            greys.append([0.4 if tless else BLENDER_DEFAULT_GREY] * 3)
        poses = np.stack(poses)
        out = render_views(meshes, poses, args.size, greys)
        dropped = out["dropped"].cpu().numpy()
        for o, obj_id in enumerate(ids):
            if dropped[o]:
                print(f"=> WARNING: obj {obj_id}: {dropped[o]} triangle views dropped (vertex behind the camera or outside the guard band)")
            tdir = write_views(out, o, os.path.join(args.output_dir, args.dataset_name, f'obj_{int(obj_id):06d}'), to_metres(poses[o]))
            print(f"=> obj {obj_id}: {poses.shape[1]} templates written to {tdir}")
    return 0


if __name__ == "__main__":
    main()
