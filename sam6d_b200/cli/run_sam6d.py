"""SAM-6D's demo.sh in one process: render the CAD templates, segment and score the frame (ISM), estimate the poses (PEM),
with every model built once and no file between the stages (sam6d_b200/pipeline.py: SAM6D).

    python -m sam6d_b200.cli.run_sam6d --cad_path obj.ply --rgb_path rgb.png --depth_path depth.png --cam_path camera.json \\
        --output_dir OUT [--segmentor_model sam|fastsam [--fastsam_model FastSAM-x|FastSAM-s]] [--checkpoint_dir checkpoints --checkpoint sam-6d-pem-base.pth]

With several CAD models (--cad_path a.ply b.ply ... [--obj_ids 1 5 ...]) the frame runs through SAM6D.detect_objects: the ISM's
multi-object post-processing (size filter, per-object NMS), records with category_id = the object's id (default 1, 2, ...),
and one PEM batch across the objects; vis_pem.png draws each object's best pose with that object's points.

--rendering_type pbr --pbr_root DATASET [--pbr_split train_pbr] takes the ISM references from the BOP PBR split DATASET/train_pbr
instead of GPU renders (the reference's default onboarding_config.rendering_type; sam6d_b200/pbr.py).  It needs --obj_ids, the
BOP ids of the CAD models, and --pose_distribution all.

Writes what the chained CLIs write as results: $OUT/sam6d_results/detection_ism.json, detection_pem.json and vis_pem.png,
with the same records.  It does not write the template files ($OUT/templates/*) nor detection_ism.npz: the npz is an
intermediate of the reference that nothing downstream reads, and writing it would copy every dense proposal mask to the
host, which the device-side RLE hand-off exists to avoid.  Random draws use numpy's global RNG in the chained CLIs' order, so
`np.random.seed(s)` before this CLI gives what `np.random.seed(s)` before the ISM CLI gives the chain."""
import argparse
import json
import os
import sys

from . import ism_run_inference_custom as ism_cli
from . import pem_run_inference_custom as pem_cli


class _OneOrSeveral(argparse.Action):
    """nargs="+" that stores one value as itself and several as a list"""

    def __call__(self, parser, namespace, values, option_string=None):
        setattr(namespace, self.dest, values[0] if len(values) == 1 else list(values))


def get_parser():
    ap = argparse.ArgumentParser(description="SAM-6D: templates -> ISM -> PEM in one process")
    ap.add_argument("--output_dir", required=True, help="Path to root directory of the output")
    ap.add_argument("--cad_path", required=True, nargs="+", action=_OneOrSeveral, help="Path to CAD(mm); several for several objects")
    ap.add_argument("--obj_ids", type=int, nargs="+", default=None, help="category ids of the CAD models (default 1..O)")
    ap.add_argument("--rgb_path", required=True, help="Path to RGB image")
    ap.add_argument("--depth_path", required=True, help="Path to Depth image(mm)")
    ap.add_argument("--cam_path", required=True, help="Path to camera information")
    add_model_args(ap)
    return ap


def add_model_args(ap, frames: bool = True):
    """the model and pose options of run_sam6d, track_sam6d and run_bop.  frames=False leaves out --det_score_thresh and
    --pbr_root: run_bop filters detections by the BOP rule and takes the PBR split from its dataset"""
    ap.add_argument("--template_size", default=512, type=int, help="template width and height in pixels (render_custom_templates --size)")
    # the ISM CLI's options
    ap.add_argument("--segmentor_model", default="sam", choices=("sam", "fastsam"), help="The segmentor model in ISM")
    ap.add_argument("--stability_score_thresh", default=0.97, type=float, help="stability_score_thresh of SAM")
    ap.add_argument("--checkpoint_dir", default=None, help="the ISM CLI's --checkpoint_dir (SAM / FastSAM and DINOv2 weights)")
    ap.add_argument("--sam_model_type", default="vit_h", choices=("vit_h", "vit_l", "vit_b"))
    ap.add_argument("--fastsam_model", default="FastSAM-x", choices=tuple(ism_cli.FASTSAM_MODELS))
    ap.add_argument("--dinov2_model", default="dinov2_vitl14", choices=("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14"))
    ap.add_argument("--points_per_side", default=32, type=int)
    ap.add_argument("--pred_iou_thresh", default=0.88, type=float)
    ap.add_argument("--confidence_thresh", default=ism_cli.CONFIDENCE_THRESH, type=float, help="semantic-score threshold")
    ap.add_argument("--aggregation_function", default="avg_5", choices=("mean", "median", "max", "avg_5"),
                    help="matching_config.aggregation_function of the semantic score")
    ap.add_argument("--level_templates", default=0, type=int, choices=(0, 1, 2),
                    help="the ISM's views (onboarding_config): 0 / 1 / 2 = 42 / 162 / 642; the PEM keeps the 42 level-0 views")
    ap.add_argument("--pose_distribution", default="all", choices=("all", "upper"),
                    help="onboarding_config.pose_distribution: all, or upper (cameras with z >= 0)")
    ap.add_argument("--rendering_type", default="pyrender", choices=("pyrender", "pbr"),
                    help="onboarding_config.rendering_type: ISM references rendered from the CAD models, or frames of a BOP PBR split")
    ap.add_argument("--pbr_split", default="train_pbr", help="with --rendering_type pbr: the split whose frames become the references")
    # the PEM CLI's options
    ap.add_argument("--checkpoint", default=None, help="sam-6d-pem-base.pth (default: the PEM CLI's)")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--random_weights", action="store_true", help="seeded random weights when no checkpoints exist (plumbing runs)")
    pem_cli.add_pose_args(ap)
    if frames:
        ap.add_argument("--pbr_root", default=None, help="with --rendering_type pbr: the BOP dataset directory (holding --pbr_split)")
        ap.add_argument("--det_score_thresh", default=0.2, type=float, help="The score threshold of detection")


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    pem_cli.check_pose_args(ap, args)
    if args.rendering_type == "pbr" and (args.obj_ids is None or args.pbr_root is None):
        ap.error("--rendering_type pbr needs --pbr_root and --obj_ids (the BOP ids of the CAD models)")
    sam6d = build_sam6d(args, pbr_root=args.pbr_root, det_score_thresh=args.det_score_thresh)
    multi = isinstance(args.cad_path, list)
    n_cad = len(args.cad_path) if multi else 1
    if args.obj_ids is not None and len(args.obj_ids) != n_cad:
        raise SystemExit(f"--obj_ids: {len(args.obj_ids)} ids for {n_cad} CAD models")
    if multi:
        obj = sam6d.onboard_objects(args.cad_path, obj_ids=args.obj_ids, template_size=args.template_size,
                                    symmetries=pem_cli.symmetry_option(args))
    else:
        obj = sam6d.onboard(args.cad_path, template_size=args.template_size,
                            obj_id=args.obj_ids[0] if args.rendering_type == "pbr" else None, symmetries=pem_cli.symmetry_option(args))
    cam = json.load(open(args.cam_path))
    rgb = pem_cli.load_im(args.rgb_path).astype("uint8")
    run = sam6d.detect_objects if multi else sam6d
    res = run(rgb, pem_cli.load_im(args.depth_path), cam["cam_K"], cam["depth_scale"], obj)
    out_dir = os.path.join(args.output_dir, "sam6d_results")
    os.makedirs(out_dir, exist_ok=True)
    json.dump(res.ism, open(os.path.join(out_dir, "detection_ism.json"), "w"))
    with open(os.path.join(out_dir, "detection_pem.json"), "w") as f:
        json.dump(res.pem, f)
    if res.reason is not None:
        print(f"=> {res.reason}")
    print(f"=> {len(res.ism)} ISM detections, {len(res.pem)} poses written to {out_dir}")
    if res.pem:
        pem_cli.write_vis(os.path.join(out_dir, "vis_pem.png"), res.frame, cam["cam_K"])
    return 0


def build_sam6d(args, pbr_root=None, **kw):
    """the SAM6D of add_model_args' options; pbr_root: the BOP dataset of --rendering_type pbr; kw: SAM6D's other arguments"""
    from ..pipeline import SAM6D
    return SAM6D(segmentor=args.segmentor_model, sam_model_type=args.sam_model_type, fastsam_model=args.fastsam_model,
                 dinov2_model=args.dinov2_model,
                 checkpoint_dir=args.checkpoint_dir, checkpoint=args.checkpoint, random_weights=args.random_weights,
                 stability_score_thresh=args.stability_score_thresh, pred_iou_thresh=args.pred_iou_thresh,
                 points_per_side=args.points_per_side, confidence_thresh=args.confidence_thresh,
                 precision=args.precision, level_templates=args.level_templates,
                 pose_distribution=args.pose_distribution, aggregation_function=args.aggregation_function,
                 rendering_type=args.rendering_type, pbr_root=pbr_root, pbr_split=args.pbr_split,
                 icp_iters=args.icp_iters, verify=args.verify, verify_tau=args.verify_tau, pem_hypotheses=args.pem_hypotheses,
                 hyp_min_angle=args.hyp_min_angle, hyp_min_dist=args.hyp_min_dist, **kw)


if __name__ == "__main__":
    sys.exit(main())
