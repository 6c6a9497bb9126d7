"""Write a BOP models_info.json for CAD models in mm, computed on the GPU (not in the reference; sam6d_b200/symmetry.py):

    python -m sam6d_b200.cli.make_models_info --cad_path a.ply b.ply --obj_ids 1 2 --output models_info.json
    python -m sam6d_b200.cli.make_models_info --models_dir DIR --output DIR/models_info.json     # every DIR/obj_*.ply

Each entry holds diameter, min_x/y/z, size_x/y/z and the symmetries find_symmetries finds (symmetries_discrete,
symmetries_continuous), in BOP's format, so bop.load_objects, render_bop_templates and eval_bop read the file unchanged."""
import argparse
import glob
import json
import os
import sys


def get_parser():
    ap = argparse.ArgumentParser(description="models_info.json (diameter, bounding box, symmetries) of CAD models in mm")
    ap.add_argument("--cad_path", nargs="+", default=None, help="CAD models (PLY, mm)")
    ap.add_argument("--obj_ids", type=int, nargs="+", default=None, help="the object id of each --cad_path (default 1..N)")
    ap.add_argument("--models_dir", default=None, help="a BOP models folder: every obj_XXXXXX.ply, ids from the file names")
    ap.add_argument("--output", required=True, help="the models_info.json to write")
    ap.add_argument("--geo_tol", type=float, default=None, help="surface tolerance over the diameter (default symmetry.GEO_TOL)")
    ap.add_argument("--color_tol", type=float, default=None, help="colour tolerance in [0, 1] (default symmetry.COLOR_TOL)")
    ap.add_argument("--slack", type=float, default=None, help="agreement slack over the query count (default symmetry.SLACK)")
    ap.add_argument("--geometry_only", action="store_true", help="ignore vertex colours and textures")
    return ap


def models(ap, args):
    """-> [(obj_id, ply path)] of the arguments; ap.error on a bad combination"""
    if (args.cad_path is None) == (args.models_dir is None):
        ap.error("give either --cad_path (with optional --obj_ids) or --models_dir")
    if args.models_dir is not None:
        if args.obj_ids is not None:
            ap.error("--obj_ids goes with --cad_path; --models_dir takes the ids from the obj_XXXXXX.ply names")
        paths = sorted(glob.glob(os.path.join(args.models_dir, "obj_*.ply")))
        if not paths:
            ap.error(f"no obj_*.ply in {args.models_dir}")
        try:
            return [(int(os.path.basename(p)[4:-4]), p) for p in paths]
        except ValueError:
            ap.error(f"{args.models_dir}: model files are named obj_<id>.ply")
    ids = list(range(1, len(args.cad_path) + 1)) if args.obj_ids is None else args.obj_ids
    if len(ids) != len(args.cad_path) or len(set(ids)) != len(ids):
        ap.error(f"--obj_ids: {len(args.cad_path)} CAD models need {len(args.cad_path)} distinct ids, got {ids}")
    for p in args.cad_path:
        if not os.path.isfile(p):
            ap.error(f"no CAD model {p}")
    return list(zip(ids, args.cad_path))


def main(argv=None):
    ap = get_parser()
    args = ap.parse_args(argv)
    todo = models(ap, args)
    from .. import meshio, symmetry
    kw = dict(use_appearance=not args.geometry_only)
    for k in ("geo_tol", "color_tol", "slack"):
        if getattr(args, k) is not None:
            kw[k] = getattr(args, k)
    try:
        symmetry._check_args(kw.get("geo_tol", symmetry.GEO_TOL), kw.get("color_tol", symmetry.COLOR_TOL), kw.get("slack", symmetry.SLACK))
    except ValueError as e:
        ap.error(str(e))
    info = {}
    for obj_id, path in todo:
        info[str(obj_id)] = symmetry.models_info_entry(meshio.load_ply_mesh(path), **kw)
        e = info[str(obj_id)]
        print(f"=> obj {obj_id}: diameter {e['diameter']:.3f}, {len(e.get('symmetries_discrete', []))} discrete and "
              f"{len(e.get('symmetries_continuous', []))} continuous symmetries")
    os.makedirs(os.path.dirname(os.path.abspath(args.output)), exist_ok=True)
    with open(args.output, "w") as fh:
        json.dump(info, fh, indent=2)
    print(f"=> {len(info)} entries written to {args.output}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
