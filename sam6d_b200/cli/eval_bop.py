"""Score a BOP results CSV (cli/run_bop's result_<dataset>.csv) with the BOP19 pose-task metrics (sam6d_b200/bop_eval.py).

    python -m sam6d_b200.cli.eval_bop --bop_root BOP --dataset_name ycbv --result_csv out/result_ycbv.csv --output_dir out \\
        [--targets FILE] [--error_types vsd mssd mspd]

Writes OUT/scores_bop19_<dataset>.json (ARs, the recall at every threshold and the counts) and prints AR_VSD, AR_MSSD, AR_MSPD
and AR.  Ground truth, cameras and test depth come from BOP/<dataset>/<test split>, models from BOP/<dataset>/models_eval."""
import argparse
import json
import os
import sys

from .. import bop, bop_eval


def get_parser():
    ap = argparse.ArgumentParser(description="BOP19 pose scores (AR_VSD, AR_MSSD, AR_MSPD, AR) of a results CSV")
    ap.add_argument("--bop_root", required=True, help="directory holding the BOP datasets (<bop_root>/<dataset_name>)")
    ap.add_argument("--dataset_name", required=True, help="BOP dataset name, e.g. ycbv, lmo, tless")
    ap.add_argument("--result_csv", required=True, help="scene_id,im_id,obj_id,score,R,t,time lines (cli/run_bop's output)")
    ap.add_argument("--output_dir", required=True, help="where scores_bop19_<dataset_name>.json is written")
    ap.add_argument("--targets", default=None, help="targets file (default <bop_root>/<dataset_name>/test_targets_bop19.json)")
    ap.add_argument("--error_types", nargs="+", default=list(bop_eval.ERROR_TYPES), choices=bop_eval.ERROR_TYPES)
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
    if not os.path.isfile(args.result_csv):
        ap.error(f"no results file {args.result_csv}")
    error_types = tuple(dict.fromkeys(args.error_types))
    scores = bop_eval.evaluate_bop19(args.bop_root, args.dataset_name, args.result_csv, targets=targets, error_types=error_types)
    os.makedirs(args.output_dir, exist_ok=True)
    out = os.path.join(args.output_dir, f"scores_bop19_{args.dataset_name}.json")
    with open(out, "w") as fh:
        json.dump(scores, fh, indent=1)
    for e in error_types:
        print(f"AR_{e.upper()}: {scores[f'ar_{e}']:.4f}")
    print(f"AR: {scores['ar']:.4f}")
    print(f"=> {out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
