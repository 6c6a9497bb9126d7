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

from . import pem_run_inference_custom as pem_cli
from . import run_sam6d
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
    run_sam6d.add_model_args(ap, frames=False)
    return ap


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    pem_cli.check_pose_args(ap, args, models_info=True)
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
    sam6d = run_sam6d.build_sam6d(args, pbr_root=dataset_root if args.rendering_type == "pbr" else None)
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
