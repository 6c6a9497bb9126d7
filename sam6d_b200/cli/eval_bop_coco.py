"""Score an ISM result JSON (cli/run_bop's result_<dataset>.json) with the BOP detection / segmentation metrics: COCO AP and AR
(sam6d_b200/bop_eval_coco.py).

    python -m sam6d_b200.cli.eval_bop_coco --bop_root BOP --dataset_name ycbv --result_json out/result_ycbv.json --output_dir out \\
        [--targets FILE] [--iou_type segm|bbox] [--bbox_type amodal|modal]

Writes OUT/scores_bop22_coco_<iou_type>_<dataset>.json (the 12 COCO stats, AP per object, the precision and recall arrays and
the counts) and prints the 12 stats.  Ground truth and masks come from BOP/<dataset>/<test split>."""
import argparse
import json
import os
import sys

from .. import bop, bop_eval_coco


def get_parser():
    ap = argparse.ArgumentParser(description="BOP detection / segmentation scores (COCO AP and AR) of an ISM result JSON")
    ap.add_argument("--bop_root", required=True, help="directory holding the BOP datasets (<bop_root>/<dataset_name>)")
    ap.add_argument("--dataset_name", required=True, help="BOP dataset name, e.g. ycbv, lmo, tless")
    ap.add_argument("--result_json", required=True, help="detection records with uncompressed RLE masks (cli/run_bop's output)")
    ap.add_argument("--output_dir", required=True, help="where scores_bop22_coco_<iou_type>_<dataset_name>.json is written")
    ap.add_argument("--targets", default=None, help="targets file (default <bop_root>/<dataset_name>/test_targets_bop19.json)")
    ap.add_argument("--iou_type", default="segm", choices=bop_eval_coco.IOU_TYPES, help="segm: mask IoU, bbox: box IoU")
    ap.add_argument("--bbox_type", default="amodal", choices=bop_eval_coco.BBOX_TYPES,
                    help="GT boxes from the full masks (amodal) or the visible masks (modal)")
    return ap


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    dataset_root = os.path.join(args.bop_root, args.dataset_name)
    if not os.path.isdir(dataset_root):
        ap.error(f"no dataset directory {dataset_root}")
    split = os.path.join(dataset_root, bop.split_name(args.dataset_name))
    if not os.path.isdir(split):
        ap.error(f"no test split directory {split}")
    targets = args.targets or os.path.join(dataset_root, "test_targets_bop19.json")
    if not os.path.isfile(targets):
        ap.error(f"no targets file {targets}")
    if not os.path.isfile(args.result_json):
        ap.error(f"no results file {args.result_json}")
    scores = bop_eval_coco.evaluate_bop22_coco(args.bop_root, args.dataset_name, args.result_json, targets=targets,
                                               iou_type=args.iou_type, bbox_type=args.bbox_type)
    os.makedirs(args.output_dir, exist_ok=True)
    out = os.path.join(args.output_dir, f"scores_bop22_coco_{args.iou_type}_{args.dataset_name}.json")
    with open(out, "w") as fh:
        json.dump(scores, fh, indent=1)
    for name in bop_eval_coco.STAT_NAMES:
        print(f"{name}: {scores[name]:.4f}")
    print(f"=> {out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
