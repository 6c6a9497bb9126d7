"""Build a coloured object model in mm from posed RGB-D views, for objects without a CAD model (not in the reference;
sam6d_b200/fusion.py):

    python -m sam6d_b200.cli.fuse_object_model --scene_dir up down --obj_id 1 --output_ply obj.ply
    python -m sam6d_b200.cli.run_sam6d --cad_path obj.ply ...

Each --scene_dir is a scene in BOP layout: rgb/ (or gray/), depth/, mask/ or mask_visib/ (<im_id>_<gt_idx>.png),
scene_camera.json (cam_K, depth_scale) and scene_gt.json (cam_R_m2c, cam_t_m2c in mm, obj_id).  Every frame that lists
--obj_id in scene_gt.json is fused (its first instance there); frames without it are skipped and counted.  Several scenes,
such as an object's up and down onboarding sequences, give one model.  The poses are an input: they are not estimated here.

Masks: mask/ (the object's full silhouette) is preferred over mask_visib/.  Outside the mask the views carve free space; a
visible-only mask also carves the parts of the object that something else occludes, which the depth then cannot restore.
Without either folder the depth alone is fused (everything it sees becomes part of the model).

The PLY (binary, vertex colours) feeds run_sam6d --cad_path, track_sam6d and make_models_info unchanged."""
import argparse
import glob
import json
import os
import sys

import numpy as np


def get_parser():
    ap = argparse.ArgumentParser(description="fuse posed RGB-D views (BOP scene layout) into a coloured mesh in mm")
    ap.add_argument("--scene_dir", nargs="+", required=True, help="BOP-layout scene folders, fused into one model")
    ap.add_argument("--obj_id", type=int, required=True, help="the object's id in scene_gt.json")
    ap.add_argument("--output_ply", required=True, help="the PLY to write")
    ap.add_argument("--frame_step", type=int, default=1, help="fuse every n-th frame of each scene")
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--resolution", type=int, default=None, help="voxels along the longest side of the views' box (default 128)")
    g.add_argument("--voxel_size", type=float, default=None, help="voxel size in mm (instead of --resolution)")
    ap.add_argument("--trunc_voxels", type=float, default=4.0, help="truncation distance in voxels")
    ap.add_argument("--min_weight", type=int, default=1, help="views a lattice corner needs before it may carry surface")
    return ap


def _image(folder, im_id):
    """the image of im_id in folder (any extension) or None"""
    hits = sorted(glob.glob(os.path.join(folder, f"{im_id:06d}.*")))
    return hits[0] if hits else None


def scene_frames(scene_dir, obj_id, frame_step=1):
    """the frames of one BOP-layout scene that show obj_id -> (frames, skipped, mask folder or None).  frames: dicts of
    rgb, depth, mask (path or None), cam_K (3,3), depth_scale, pose (4,4) with t in mm.  Raises ValueError with the missing
    file's name."""
    def need(path):
        if not os.path.exists(path):
            raise ValueError(f"{scene_dir}: no {os.path.basename(path)}")
        return path
    with open(need(os.path.join(scene_dir, "scene_camera.json"))) as fh:
        cams = json.load(fh)
    with open(need(os.path.join(scene_dir, "scene_gt.json"))) as fh:
        gts = json.load(fh)
    rgb_dir = next((os.path.join(scene_dir, d) for d in ("rgb", "gray") if os.path.isdir(os.path.join(scene_dir, d))), None)
    if rgb_dir is None:
        raise ValueError(f"{scene_dir}: no rgb/ or gray/ folder")
    depth_dir = need(os.path.join(scene_dir, "depth"))
    mask_dir = next((os.path.join(scene_dir, d) for d in ("mask", "mask_visib") if os.path.isdir(os.path.join(scene_dir, d))), None)
    frames, skipped = [], 0
    for n, key in enumerate(sorted(gts, key=int)):
        if n % frame_step:
            continue
        im_id = int(key)
        inst = [i for i, g in enumerate(gts[key]) if int(g["obj_id"]) == obj_id]
        if not inst:
            skipped += 1
            continue
        if key not in cams:
            raise ValueError(f"{scene_dir}: image {im_id} is in scene_gt.json but not in scene_camera.json")
        g = gts[key][inst[0]]
        pose = np.eye(4)
        pose[:3, :3] = np.asarray(g["cam_R_m2c"], np.float64).reshape(3, 3)
        pose[:3, 3] = np.asarray(g["cam_t_m2c"], np.float64).reshape(3)
        rgb, depth = _image(rgb_dir, im_id), _image(depth_dir, im_id)
        if rgb is None or depth is None:
            raise ValueError(f"{scene_dir}: image {im_id} has no {'rgb' if rgb is None else 'depth'} file")
        mask = None
        if mask_dir is not None:
            mask = os.path.join(mask_dir, f"{im_id:06d}_{inst[0]:06d}.png")
            if not os.path.exists(mask):
                raise ValueError(f"{scene_dir}: no {os.path.basename(mask_dir)}/{os.path.basename(mask)}")
        frames.append(dict(rgb=rgb, depth=depth, mask=mask, cam_K=np.asarray(cams[key]["cam_K"], np.float64).reshape(3, 3),
                           depth_scale=float(cams[key].get("depth_scale", 1.0)), pose=pose))
    return frames, skipped, mask_dir


def load_views(frames):
    """decode the frames -> (rgb (T,H,W,3) u8, depth (T,H,W) f32 in mm, masks (T,H,W) u8 or None, K (T,3,3), poses (T,4,4)).
    Depth is scaled to mm per frame, since scenes may differ in depth_scale."""
    from .. import bop, pbr
    if not frames:
        raise ValueError("no frame shows the object")
    with_mask = [f["mask"] is not None for f in frames]
    if any(with_mask) and not all(with_mask):
        raise ValueError("some scenes have masks and others do not: fuse them separately or give every scene masks")
    rgb, depth, masks = [], [], []
    for f in frames:
        rgb.append(bop.decode_rgb(f["rgb"]))
        depth.append(bop.decode_depth(f["depth"]).astype(np.float32) * np.float32(f["depth_scale"]))
        if f["mask"] is not None:
            masks.append(pbr.decode_mask(f["mask"]))
    shapes = {d.shape for d in depth} | {r.shape[:2] for r in rgb} | {m.shape for m in masks}
    if len(shapes) != 1:
        raise ValueError(f"every frame must have one image size, got {sorted(shapes)}")
    return (np.stack(rgb), np.stack(depth), np.stack(masks) if masks else None, np.stack([f["cam_K"] for f in frames]),
            np.stack([f["pose"] for f in frames]))


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    if args.frame_step < 1:
        ap.error("--frame_step must be >= 1")
    if args.min_weight < 1:
        ap.error("--min_weight must be >= 1")
    if not (args.trunc_voxels > 0 and np.isfinite(args.trunc_voxels)):
        ap.error("--trunc_voxels must be finite and > 0")
    if args.resolution is not None and args.resolution < 2:
        ap.error("--resolution must be >= 2")
    if args.voxel_size is not None and not (args.voxel_size > 0 and np.isfinite(args.voxel_size)):
        ap.error("--voxel_size must be finite and > 0")
    frames, skipped, folders = [], 0, set()
    for d in args.scene_dir:
        if not os.path.isdir(d):
            ap.error(f"no scene folder {d}")
        try:
            f, s, m = scene_frames(d, args.obj_id, args.frame_step)
        except ValueError as e:
            ap.error(str(e))
        frames += f
        skipped += s
        folders.add(None if m is None else os.path.basename(m))
    print(f"=> obj {args.obj_id}: {len(frames)} frames, {skipped} skipped without it, masks from {sorted(map(str, folders))}")
    if not frames:
        ap.error(f"no frame of {args.scene_dir} shows obj_id {args.obj_id}")
    from .. import fusion, meshio
    try:
        rgb, depth, masks, K, poses = load_views(frames)
        mesh = fusion.fuse(rgb, depth, masks, K, poses, 1.0, resolution=args.resolution or fusion.DEFAULT_RESOLUTION,
                           voxel_size_mm=args.voxel_size, trunc_voxels=args.trunc_voxels, min_weight=args.min_weight)
    except ValueError as e:
        ap.error(str(e))
    if len(mesh.faces) == 0:
        ap.error("the fused volume holds no surface: check the poses, depth_scale and masks")
    os.makedirs(os.path.dirname(os.path.abspath(args.output_ply)), exist_ok=True)
    meshio.save_ply(args.output_ply, mesh)
    print(f"=> {len(mesh.vertices)} vertices, {len(mesh.faces)} faces written to {args.output_ply}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
