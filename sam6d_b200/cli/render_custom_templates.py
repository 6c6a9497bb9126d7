"""Drop-in for SAM-6D/Render/render_custom_templates.py: the 42 template views of one CAD model, rendered on the GPU in one
rasteriser call (sam6d_b200/render.py) instead of BlenderProc.  Same arguments, same files:
    $OUT/templates/rgb_i.png, mask_i.png (255 = object), xyz_i.npy (object coordinates in mm, float16),  i = 0..41
plus templates/template_poses.npy (42,4,4): the object -> camera pose of every view in the order rendered, translation in
metres, which the ISM CLI's geometric score reads.

    python -m sam6d_b200.cli.render_custom_templates --cad_path obj.ply --output_dir OUT [--colorize True --base_color 0.05]

Framing as in the reference: with --normalize the model is scaled by 1/(2r), r = max(|bbox max|, |bbox min|) of the vertices
(the reference takes r from 1024 random surface samples), and the camera is 2 units away, i.e. d = 4r in model units; without
it d = 2.  The views are sam6d_b200.render.level0_template_poses() (elevation, then azimuth ascending); --poses takes the
reference's obj_poses_level0.npy (or any (T,4,4) file whose translation is in mm for a camera 1000 mm away) to render in its
order.  Colours: --colorize paints the model in --base_color; otherwise the texture, else the vertex colours, else Blender's
default grey 0.8.  Shading is ambient + Lambert from a point light at 2.5x the camera position, not Cycles.

Denser view sets for the ISM (the reference's onboarding_config): --level_templates {0,1,2} (42 / 162 / 642 views) and
--pose_distribution {all,upper} (upper: cameras with z >= 0).  The directory then holds render.template_view_set()'s layout:
the 42 level-0 views first as rgb_0..41 (what the PEM reads, the same files as the defaults write), then the chosen set's other
views; template_poses.npy follows the same order.  The ISM CLI given the same two flags finds its views among them."""
import argparse
import os

import numpy as np
import torch

from .. import meshio, render

BLENDER_DEFAULT_GREY = 0.8


def get_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cad_path', help="The path of CAD model")
    ap.add_argument('--output_dir', help="The path to save CAD templates")
    ap.add_argument('--normalize', default=True, help="Whether to normalize CAD model or not")
    ap.add_argument('--colorize', default=False, help="Whether to colorize CAD model or not")
    ap.add_argument('--base_color', default=0.05, help="The base color used in CAD model")
    # not in the reference
    ap.add_argument('--size', type=int, default=512, help="template width and height in pixels (the reference renders 512)")
    ap.add_argument('--poses', default=None, help="(T,4,4) .npy of object -> camera poses, translation in mm at 1000 mm "
                                                  "(the reference's obj_poses_level0.npy); default: level0_template_poses()")
    return ap


def view_set_parser():
    """the view-set flags, not in the reference's argument list (get_parser): parsed from what get_parser leaves"""
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--level_templates", type=int, default=0, choices=sorted(render.VIEW_COUNTS),
                    help="onboarding_config.level_templates: 0 / 1 / 2 = 42 / 162 / 642 views")
    ap.add_argument("--pose_distribution", default="all", choices=render.POSE_DISTRIBUTIONS,
                    help="onboarding_config.pose_distribution: all, or upper (cameras with z >= 0)")
    return ap


def view_poses(distance, poses_file=None):
    """(T,4,4) float64 object -> camera poses with the camera `distance` model units from the origin"""
    return view_set(distance, poses_file)[0]


def view_set(distance, poses_file=None, level_templates=0, pose_distribution="all"):
    """-> (poses (N,4,4) float64 with the camera `distance` model units from the origin, ism_index (T,) int64):
    render.template_view_set's layout, or poses_file's views (then all of them are the ISM's, and the view set must be the
    default one)"""
    if poses_file is None:
        return render.template_view_set(level_templates, pose_distribution, distance)
    if (level_templates, pose_distribution) != (0, "all"):
        raise ValueError("--poses renders the file's views: it takes no --level_templates / --pose_distribution")
    P = np.asarray(np.load(poses_file), dtype=np.float64).reshape(-1, 4, 4).copy()
    P[:, :3, 3] *= distance / 1000.0
    return P, np.arange(len(P), dtype=np.int64)


def render_views(meshes_dev, poses, size, base_colors):
    """meshes on the device, poses (O,T,4,4) float64 in model units -> render.render()'s dict"""
    return render.render(meshes_dev, torch.from_numpy(poses.astype(np.float32)).cuda(), render.template_K(size), size, size,
                         base_color=np.asarray(base_colors, np.float32))


def write_views(out, o, tdir, poses_m):
    """views of object o of render()'s output -> rgb_i.png, mask_i.png, xyz_i.npy, template_poses.npy under tdir"""
    import cv2
    os.makedirs(tdir, exist_ok=True)
    rgb, mask, xyz = out["rgb"][o].cpu().numpy(), out["mask"][o].cpu().numpy(), out["xyz"][o].cpu().numpy()
    for i in range(len(rgb)):
        cv2.imwrite(os.path.join(tdir, f"rgb_{i}.png"), rgb[i][:, :, ::-1])          # files hold RGB as load_im reads it
        cv2.imwrite(os.path.join(tdir, f"mask_{i}.png"), mask[i])
        np.save(os.path.join(tdir, f"xyz_{i}.npy"), xyz[i])
    np.save(os.path.join(tdir, "template_poses.npy"), poses_m)
    return tdir


def to_metres(poses_mm):
    P = np.array(poses_mm, dtype=np.float64)
    P[..., :3, 3] /= 1000.0
    return P


def parse_args(argv=None):
    """get_parser()'s arguments plus view_set_parser()'s, in one namespace"""
    args, rest = get_parser().parse_known_args(argv)
    view_set_parser().parse_args(rest, namespace=args)
    return args


def main(argv=None):
    args = parse_args(argv)
    from ..pipeline import render_templates
    out, poses = render_templates(meshio.load_ply_mesh(args.cad_path), args.size, args.normalize, args.colorize, args.base_color, args.poses,
                                  args.level_templates, args.pose_distribution)
    dropped = int(out["dropped"][0])
    if dropped:
        print(f"=> WARNING: {dropped} triangle views dropped (vertex behind the camera or outside the guard band)")
    tdir = write_views(out, 0, os.path.join(args.output_dir, "templates"), to_metres(poses))
    print(f"=> {len(poses)} templates written to {tdir}")
    return 0


if __name__ == "__main__":
    main()
