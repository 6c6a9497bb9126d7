"""Track objects through an RGB-D sequence (not in the reference; sam6d_b200/track.py: Tracker): detect with SAM-6D on the
first frame, then follow each object's pose with depth and ICP, detecting again only to start or recover a track.

    python -m sam6d_b200.cli.track_sam6d --cad_path a.ply b.ply [--obj_ids 1 5] --rgb_dir RGB --depth_dir DEPTH \\
        --cam_path camera.json --output_dir OUT [run_sam6d's model options] [--track_icp_iters 10 --margin_px 16 ...]

Frames are the file names present in both --rgb_dir and --depth_dir, in sorted order; one camera.json (cam_K, depth_scale)
serves every frame.  Writes $OUT/sam6d_results/track_pem.json: a list with one {"frame": name, "records": [...]} per frame,
the records as Tracker returns them (detection_pem.json's keys plus "track" and "frames_tracked", and "track_id" with
--max_instances above 1)."""
import argparse
import json
import os
import sys

from . import pem_run_inference_custom as pem_cli
from . import run_sam6d


def get_parser():
    ap = argparse.ArgumentParser(description="SAM-6D tracking: detect, then follow each object's pose with depth")
    ap.add_argument("--cad_path", required=True, nargs="+", help="Path to CAD(mm), one per object")
    ap.add_argument("--obj_ids", type=int, nargs="+", default=None, help="category ids of the CAD models (default 1..O)")
    ap.add_argument("--rgb_dir", required=True, help="directory of the RGB frames")
    ap.add_argument("--depth_dir", required=True, help="directory of the depth frames (mm), named as the RGB frames")
    ap.add_argument("--cam_path", required=True, help="Path to camera information")
    ap.add_argument("--output_dir", required=True, help="Path to root directory of the output")
    run_sam6d.add_model_args(ap)
    # the tracker's parameters (sam6d_b200/track.py; not tuned on real video)
    ap.add_argument("--track_icp_iters", default=10, type=int, help="ICP iterations per tracked frame")
    ap.add_argument("--margin_px", default=16, type=int, help="dilation of the rendered silhouette in pixels")
    ap.add_argument("--gate_scale", default=1.5, type=float, help="gate radius over the object's radius about its centroid")
    ap.add_argument("--min_inlier_fraction", default=0.5, type=float, help="a track with fewer ICP inliers is lost")
    ap.add_argument("--max_rms_m", default=0.005, type=float, help="a track with a larger ICP RMS (metres) is lost")
    ap.add_argument("--redetect_interval", default=30, type=int, help="frames without detection before detecting again")
    ap.add_argument("--max_instances", default=1, type=int, help="tracks per object (copies of one object in the scene)")
    ap.add_argument("--start_score", default=0.3, type=float, help="least PEM score that starts an object's second and later tracks")
    ap.add_argument("--assoc_scale", default=0.5, type=float,
                    help="centroid distance, over the object's radius, within which two tracks of one object are one copy")
    return ap


def frame_pairs(rgb_dir: str, depth_dir: str):
    """the file names present in both directories, sorted"""
    return sorted(set(os.listdir(rgb_dir)) & set(os.listdir(depth_dir)))


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    pem_cli.check_pose_args(ap, args)
    if args.rendering_type == "pbr" and (args.obj_ids is None or args.pbr_root is None):
        ap.error("--rendering_type pbr needs --pbr_root and --obj_ids (the BOP ids of the CAD models)")
    if args.obj_ids is not None and len(args.obj_ids) != len(args.cad_path):
        raise SystemExit(f"--obj_ids: {len(args.obj_ids)} ids for {len(args.cad_path)} CAD models")
    names = frame_pairs(args.rgb_dir, args.depth_dir)
    if not names:
        raise SystemExit(f"no frame is named the same in {args.rgb_dir} and {args.depth_dir}")
    from ..track import Tracker
    sam6d = run_sam6d.build_sam6d(args, pbr_root=args.pbr_root, det_score_thresh=args.det_score_thresh)
    objs = sam6d.onboard_objects(args.cad_path, obj_ids=args.obj_ids, template_size=args.template_size,
                                 symmetries=pem_cli.symmetry_option(args))
    tracker = Tracker(sam6d, objs, args.cad_path, track_icp_iters=args.track_icp_iters, margin_px=args.margin_px,
                      gate_scale=args.gate_scale, min_inlier_fraction=args.min_inlier_fraction, max_rms_m=args.max_rms_m,
                      redetect_interval=args.redetect_interval, max_instances=args.max_instances, start_score=args.start_score,
                      assoc_scale=args.assoc_scale)
    cam = json.load(open(args.cam_path))
    out = []
    for name in names:
        rgb = pem_cli.load_im(os.path.join(args.rgb_dir, name)).astype("uint8")
        res = tracker(rgb, pem_cli.load_im(os.path.join(args.depth_dir, name)), cam["cam_K"], cam["depth_scale"])
        out.append({"frame": name, "records": res.records})
        print(f"=> {name}: {' '.join(res.state)}{' (detection)' if res.detection is not None else ''}")
    out_dir = os.path.join(args.output_dir, "sam6d_results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "track_pem.json"), "w") as f:
        json.dump(out, f)
    print(f"=> {len(out)} frames written to {out_dir}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
