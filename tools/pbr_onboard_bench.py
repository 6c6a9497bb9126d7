"""tools/pbr_onboard_bench.py -- time SAM6D.onboard_objects with rendering_type "pbr" and its stages on the GPU.

    python tools/pbr_onboard_bench.py [--out pbr_onboard_bench.json]

A seeded BOP-like split is synthesised in a temporary directory: 640 x 480 JPEG frames (BOP's train_pbr format), 21 objects, each
frame showing 8 of them with 8-bit visible masks.  For O = 1 / 8 / 21 objects at level 0 / 1 it prints, each on its own line,
the seconds of: scan (pbr.scan_split), selection (pbr.select_references), decode (PIL, frames and masks), crop kernel
(sam6d_pbr_reference_crops, CUDA events), crop call (upload + kernel), descriptors (DINOv2 ViT-L/14 on the crops), and the
whole onboard_objects call (which also renders the PEM's 42 views per object).  The card's name and power limit are printed
and stored with the numbers.  Seeded random weights: the timings do not depend on the weights."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_OBJ = 21


def make_split(root, scenes=10, frames_per_scene=60, per_frame=8, seed=0):
    from PIL import Image
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:480, 0:640]
    for s in range(scenes):
        d = os.path.join(root, "train_pbr", f"{s:06d}")
        os.makedirs(os.path.join(d, "rgb"))
        os.makedirs(os.path.join(d, "mask_visib"))
        gt, info = {}, {}
        for f in range(frames_per_scene):
            img = rs.randint(0, 256, (480 // 8, 640 // 8, 3)).astype(np.uint8).repeat(8, 0).repeat(8, 1)
            Image.fromarray(img).save(os.path.join(d, "rgb", f"{f:06d}.jpg"), quality=95)
            objs = rs.choice(np.arange(1, N_OBJ + 1), per_frame, replace=False)
            gt[str(f)], info[str(f)] = [], []
            for i, o in enumerate(objs):
                q = rs.normal(size=4)
                w, x, y, z = q / np.linalg.norm(q)
                R = [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w), 1 - 2 * (x * x + z * z),
                     2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]
                gt[str(f)].append({"cam_R_m2c": R, "cam_t_m2c": [0.0, 0.0, 800.0], "obj_id": int(o)})
                info[str(f)].append({"visib_fract": float(rs.uniform(0.7, 1.0))})
                cx, cy, ax, ay = rs.uniform(100, 540), rs.uniform(80, 400), rs.uniform(30, 120), rs.uniform(30, 120)
                m = ((((xx - cx) / ax) ** 2 + ((yy - cy) / ay) ** 2) <= 1).astype(np.uint8) * 255
                Image.fromarray(m).save(os.path.join(d, "mask_visib", f"{f:06d}_{i:06d}.png"))
        json.dump(gt, open(os.path.join(d, "scene_gt.json"), "w"))
        json.dump(info, open(os.path.join(d, "scene_gt_info.json"), "w"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed, without the card line
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--objects", type=int, nargs="+", default=[1, 8, 21])
    ap.add_argument("--levels", type=int, nargs="+", default=[0, 1])
    args = ap.parse_args()
    import torch
    from sam6d_b200 import _lib, meshio, pbr, render
    from sam6d_b200.pipeline import SAM6D
    assert torch.cuda.is_available(), "the bench times the GPU"
    gpu = card()
    print(f"card, power limit: {gpu}")
    results = {"card": gpu, "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        make_split(tmp)
        print(f"synthetic split written in {time.perf_counter() - t0:.1f} s")
        verts = np.array([[x, y, z] for x in (-50, 50) for y in (-40, 40) for z in (-30, 30)], np.float32)
        faces = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                          [1, 5, 7], [1, 7, 3]], np.int64)
        mesh = meshio.Mesh(vertices=verts, faces=faces, colors=np.full((8, 3), 128, np.uint8))
        for level in args.levels:
            model = SAM6D(segmentor="fastsam", random_weights=True, rendering_type="pbr", pbr_root=tmp, level_templates=level)
            union, index = render.template_view_set(level, "all")
            views = union[index]
            for run, O in enumerate([1] + args.objects):      # run 0 warms up (module loads, allocator) and is not reported
                ids = list(range(1, O + 1))
                st = {}
                t = time.perf_counter()
                rows = pbr.scan_split(tmp)
                st["scan"] = time.perf_counter() - t
                t = time.perf_counter()
                sel = pbr.select_references(rows, ids, views, np.random.RandomState(0))
                st["selection"] = time.perf_counter() - t
                _lib.time_kernel("sam6d_pbr_reference_crops")
                pbr.reference_features(model.desc, rows, sel, model.device, timings=st)
                st["crop_kernel"] = sum(a.elapsed_time(b) for a, b in _lib.timed_events("sam6d_pbr_reference_crops")) / 1e3
                _lib.time_kernel("sam6d_pbr_reference_crops", False)
                st["crop_call"] = st.pop("crop")
                torch.cuda.synchronize()
                t = time.perf_counter()
                model.onboard_objects([mesh] * O, obj_ids=ids, template_size=512, rng=np.random.RandomState(0))
                torch.cuda.synchronize()
                st["onboard_objects"] = time.perf_counter() - t
                model._pbr_rows = None
                if run == 0:
                    continue
                rec = {"objects": O, "level": level, "templates": int(sel.size), "distinct_rows": int(len(np.unique(sel))),
                       "seconds": {k: round(v, 4) for k, v in st.items()}}
                results["runs"].append(rec)
                print(f"O={O} level={level}: {rec['templates']} references, {rec['distinct_rows']} distinct rows")
                for k in ("scan", "selection", "decode", "crop_kernel", "crop_call", "descriptors", "onboard_objects"):
                    print(f"  {k:16s} {st[k]:8.3f} s")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
