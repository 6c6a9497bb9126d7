"""SAM-6D over a BOP test split in one process: the ISM's run_inference.py (result_<dataset>.json) and the PEM's test_bop.py
(result_<dataset>.csv, the file the BOP toolkit scores), with every model built once (SAM6D.run_bop_ism / run_bop_pem).

    python -m sam6d_b200.cli.run_bop --bop_root BOP --dataset_name ycbv --template_dir BOP-Templates --output_dir OUT \\
        [--stage ism|pem|both] [--detections FILE] [--max_frames N] [the ISM options of run_sam6d]

BOP/<dataset>/{test or test_primesense, models or models_cad} is the dataset, BOP-Templates/<dataset>/obj_XXXXXX the PEM's
template views (render_bop_templates).  --stage ism writes OUT/result_<dataset>.json; --stage pem reads --detections (any
detection JSON with uncompressed RLE, default OUT/result_<dataset>.json) and writes OUT/result_<dataset>.csv; both (the
default) runs the two.  The per-frame npz and runtime files of the reference's ISM are not written: nothing downstream reads
them.  Random draws use numpy's global RNG (np.random.seed before main() fixes them)."""
import argparse
import os
import sys

from . import ism_run_inference_custom as ism_cli
from . import pem_run_inference_custom as pem_cli
from .. import bop


def get_parser():
    ap = argparse.ArgumentParser(description="SAM-6D on a BOP test split: ISM detections and PEM poses in BOP format")
    ap.add_argument("--bop_root", required=True, help="directory holding the BOP datasets (<bop_root>/<dataset_name>)")
    ap.add_argument("--dataset_name", required=True, help="BOP dataset name, e.g. ycbv, lmo, tless")
    ap.add_argument("--template_dir", default=None, help="the PEM's template directory (<template_dir>/<dataset_name>/obj_XXXXXX)")
    ap.add_argument("--output_dir", required=True, help="where result_<dataset_name>.json / .csv are written")
    ap.add_argument("--stage", default="both", choices=("ism", "pem", "both"))
    ap.add_argument("--detections", default=None, help="--stage pem: the detection JSON (default OUT/result_<dataset_name>.json)")
    ap.add_argument("--max_frames", default=None, type=int, help="only the first N frames (ISM) / images (PEM)")
    ap.add_argument("--template_size", default=512, type=int, help="ISM onboarding render size in pixels")
    ap.add_argument("--segmentor_model", default="sam", choices=("sam", "fastsam"), help="The segmentor model in ISM")
    ap.add_argument("--stability_score_thresh", default=0.97, type=float, help="stability_score_thresh of SAM")
    ap.add_argument("--checkpoint_dir", default=None, help="the ISM's checkpoints (SAM / FastSAM and DINOv2 weights)")
    ap.add_argument("--sam_model_type", default="vit_h", choices=("vit_h", "vit_l", "vit_b"))
    ap.add_argument("--fastsam_model", default="FastSAM-x", choices=tuple(ism_cli.FASTSAM_MODELS))
    ap.add_argument("--dinov2_model", default="dinov2_vitl14", choices=("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14"))
    ap.add_argument("--points_per_side", default=32, type=int)
    ap.add_argument("--pred_iou_thresh", default=0.88, type=float)
    ap.add_argument("--confidence_thresh", default=ism_cli.CONFIDENCE_THRESH, type=float, help="semantic-score threshold")
    ap.add_argument("--aggregation_function", default="avg_5", choices=("mean", "median", "max", "avg_5"))
    ap.add_argument("--level_templates", default=0, type=int, choices=(0, 1, 2))
    ap.add_argument("--pose_distribution", default="all", choices=("all", "upper"))
    ap.add_argument("--rendering_type", default="pyrender", choices=("pyrender", "pbr"),
                    help="ISM references rendered from the CAD models, or frames of the dataset's own --pbr_split")
    ap.add_argument("--pbr_split", default="train_pbr", help="with --rendering_type pbr: the split whose frames become the references")
    ap.add_argument("--checkpoint", default=None, help="sam-6d-pem-base.pth")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--random_weights", action="store_true", help="seeded random weights when no checkpoints exist (plumbing runs)")
    # not in the reference: refine each PEM pose against the observed depth (pipeline.icp_refine_out)
    ap.add_argument("--icp_iters", default=0, type=int, help="point-to-plane ICP iterations per PEM pose (0: off)")
    # not in the reference: rescore each reported pose by its agreement with the observed depth (pipeline.verify_out)
    ap.add_argument("--verify", action="store_true", help="render every pose and multiply its score by its depth agreement")
    ap.add_argument("--verify_tau", default=0.1, type=float, help="--verify's depth tolerance over the object's radius")
    pem_cli.add_hypothesis_args(ap)
    return ap


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    pem_cli.check_hypothesis_args(ap, args, models_info=True)
    if args.stage in ("pem", "both") and args.template_dir is None:
        ap.error(f"--stage {args.stage} needs --template_dir (the PEM's template views)")
    if args.stage == "both" and args.detections is not None:
        ap.error("--detections is read by --stage pem; --stage both uses the ISM's own result")
    if args.max_frames is not None and args.max_frames < 1:
        ap.error("--max_frames must be at least 1")
    dataset_root = os.path.join(args.bop_root, args.dataset_name)
    if not os.path.isdir(dataset_root):
        ap.error(f"no dataset directory {dataset_root}")
    detections = args.detections or os.path.join(args.output_dir, f"result_{args.dataset_name}.json")
    if args.stage == "pem" and not os.path.isfile(detections):
        ap.error(f"--stage pem: no detection file {detections}")
    from ..pipeline import SAM6D
    sam6d = SAM6D(segmentor=args.segmentor_model, sam_model_type=args.sam_model_type, fastsam_model=args.fastsam_model,
                  dinov2_model=args.dinov2_model, checkpoint_dir=args.checkpoint_dir, checkpoint=args.checkpoint,
                  random_weights=args.random_weights, stability_score_thresh=args.stability_score_thresh,
                  pred_iou_thresh=args.pred_iou_thresh, points_per_side=args.points_per_side, confidence_thresh=args.confidence_thresh,
                  precision=args.precision, level_templates=args.level_templates, pose_distribution=args.pose_distribution,
                  aggregation_function=args.aggregation_function, rendering_type=args.rendering_type,
                  pbr_root=dataset_root if args.rendering_type == "pbr" else None, pbr_split=args.pbr_split,
                  icp_iters=args.icp_iters, verify=args.verify, verify_tau=args.verify_tau, pem_hypotheses=args.pem_hypotheses,
                  hyp_min_angle=args.hyp_min_angle, hyp_min_dist=args.hyp_min_dist)
    os.makedirs(args.output_dir, exist_ok=True)
    if args.stage in ("ism", "both"):
        objects = sam6d.onboard_bop(args.bop_root, args.dataset_name, template_size=args.template_size)
        recs = sam6d.run_bop_ism(args.bop_root, args.dataset_name, objects, detections, max_frames=args.max_frames)
        del objects
        print(f"=> {len(recs)} detections written to {detections}")
    if args.stage in ("pem", "both"):
        out = os.path.join(args.output_dir, f"result_{args.dataset_name}.csv")
        lines = sam6d.run_bop_pem(detections, args.bop_root, args.dataset_name, args.template_dir, out, max_frames=args.max_frames,
                                  symmetries=pem_cli.symmetry_option(args))
        print(f"=> {len(lines)} poses written to {out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
