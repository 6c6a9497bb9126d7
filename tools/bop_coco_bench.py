"""Time BOP detection / segmentation scoring (sam6d_b200/bop_eval_coco.py) per stage on a synthetic split, and the float64 oracle
(oracle/bop_coco_oracle.py) per image on a few of its images.

    python tools/bop_coco_bench.py [--images 300] [--oracle_images 3] [--out DIR]

The split: 640 x 480 images with 8 GT instances each (overlapping ellipses and boxes of 4 objects, visible masks cut by the
instances before them) and 100 detections per image across the 4 objects (RLEs of shifted GT masks and false positives).
Stages of the second of two evaluate_bop22_coco runs (segm, amodal): PNG decoding of the masks, packing (pack_u8 + pack_rle
with their uploads), the pair-count kernel (with the pair upload and the count download), matching and accumulation; the three
kernels alone by CUDA events around their C calls.  Prints the card's name and power limit, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def write_split(root, n_images, H=480, W=640, n_gt=8, n_det=100, seed=0):
    from PIL import Image
    from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle
    rng = np.random.RandomState(seed)
    ds = os.path.join(root, "synth")
    y, x = np.mgrid[:H, :W]
    scenes, targets, recs = {}, [], []
    for i in range(n_images):
        s, im = 1 + i // 100, i % 100
        sdir = os.path.join(ds, "test", f"{s:06d}")
        if s not in scenes:
            for sub in ("rgb", "mask", "mask_visib"):
                os.makedirs(os.path.join(sdir, sub), exist_ok=True)
            scenes[s] = ({}, {}, {})
        Image.fromarray(np.zeros((H, W, 3), np.uint8)).save(os.path.join(sdir, "rgb", f"{im:06d}.png"))
        gt, info, cam = scenes[s]
        gt[str(im)], info[str(im)] = [], []
        cam[str(im)] = {"cam_K": [600.0, 0, 319.5, 0, 600.0, 239.5, 0, 0, 1], "depth_scale": 1.0}
        occl = np.zeros((H, W), bool)
        vis_masks = []
        for k in range(n_gt):
            o = 1 + k % 4
            cy, cx = rng.uniform(0.1, 0.9) * H, rng.uniform(0.1, 0.9) * W
            ry, rx = rng.uniform(0.02, 0.2) * H, rng.uniform(0.02, 0.2) * W
            full = (((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 <= 1.0) if k % 2 == 0 else \
                ((np.abs(y - cy) <= ry) & (np.abs(x - cx) <= rx))
            vis = full & ~occl
            occl |= full
            Image.fromarray((vis * 255).astype(np.uint8)).save(os.path.join(sdir, "mask_visib", f"{im:06d}_{k:06d}.png"))
            Image.fromarray((full * 255).astype(np.uint8)).save(os.path.join(sdir, "mask", f"{im:06d}_{k:06d}.png"))
            gt[str(im)].append({"cam_R_m2c": [1, 0, 0, 0, 1, 0, 0, 0, 1], "cam_t_m2c": [0, 0, 500], "obj_id": o})
            vf = float(vis.sum()) / max(1.0, float(full.sum()))
            info[str(im)].append({"visib_fract": vf})
            vis_masks.append((o, vis))
        targets += [{"scene_id": s, "im_id": im, "obj_id": o, "inst_count": 2} for o in range(1, 5)]
        for d in range(n_det):
            if d < n_det - 4:
                o, m = vis_masks[d % n_gt]
                m = np.roll(m, (rng.randint(-6, 7), rng.randint(-6, 7)), axis=(0, 1))
            else:
                o, m = 1 + d % 4, np.roll(vis_masks[(d + 1) % n_gt][1], (H // 3, W // 3), axis=(0, 1))
            ys, xs = np.nonzero(m)
            bb = [float(xs.min()), float(ys.min()), float(xs.max() - xs.min() + 1), float(ys.max() - ys.min() + 1)] if len(xs) else [0.0] * 4
            recs.append({"scene_id": s, "image_id": im, "category_id": o, "score": float(rng.rand()), "bbox": bb, "time": 0.1,
                         "segmentation": mask_to_rle(m.astype(np.uint8))})
    for s, (gt, info, cam) in scenes.items():
        sdir = os.path.join(ds, "test", f"{s:06d}")
        for name, obj in (("scene_gt", gt), ("scene_gt_info", info), ("scene_camera", cam)):
            with open(os.path.join(sdir, f"{name}.json"), "w") as fh:
                json.dump(obj, fh)
    with open(os.path.join(ds, "test_targets_bop19.json"), "w") as fh:
        json.dump(targets, fh)
    path = os.path.join(root, "result_synth.json")
    with open(path, "w") as fh:
        json.dump(recs, fh)
    return path, targets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=300)
    ap.add_argument("--oracle_images", type=int, default=3, help="images the float64 oracle scores on the host (timed per image)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from oracle import bop_coco_oracle as bco
    from sam6d_b200 import _lib, bop_eval_coco as bc
    print(f"[bop_coco_bench] card: {card()}")
    work = tempfile.mkdtemp(prefix="bop_coco_bench_")
    t0 = time.perf_counter()
    res, targets = write_split(work, args.images)
    t_split = time.perf_counter() - t0

    t0 = time.perf_counter()
    bc.evaluate_bop22_coco(work, "synth", res)
    torch.cuda.synchronize()
    t_first = time.perf_counter() - t0
    names = ("sam6d_bop_pack_u8", "sam6d_bop_pack_rle", "sam6d_bop_mask_pair_counts")
    for n in names:
        _lib.time_kernel(n)
    timings = {}
    t0 = time.perf_counter()
    scores = bc.evaluate_bop22_coco(work, "synth", res, timings=timings)
    torch.cuda.synchronize()
    t_eval = time.perf_counter() - t0
    kern = {n: sum(a.elapsed_time(b) for a, b in _lib.timed_events(n)) for n in names}
    calls = {n: len(_lib.timed_events(n)) for n in names}
    for n in names:
        _lib.time_kernel(n, False)
    t0 = time.perf_counter()
    bb = bc.evaluate_bop22_coco(work, "synth", res, iou_type="bbox")
    t_bbox = time.perf_counter() - t0

    # the oracle on the first few images
    sub = sorted({(t["scene_id"], t["im_id"]) for t in targets})[:args.oracle_images]
    tfile = os.path.join(work, "targets_oracle.json")
    with open(tfile, "w") as fh:
        json.dump([t for t in targets if (t["scene_id"], t["im_id"]) in sub], fh)
    t0 = time.perf_counter()
    want = bco.evaluate(work, "synth", res, targets=tfile)
    t_oracle = (time.perf_counter() - t0) / len(sub)
    got = bc.evaluate_bop22_coco(work, "synth", res, targets=tfile)
    same = bool(np.array_equal(np.array(got["precision"]), want["precision"]) and np.array_equal(np.array(got["recall"]), want["recall"]))

    rec = dict(card=card(), images=args.images, detections=scores["n_detections"], gt=scores["n_gt"], pairs=scores["n_pairs"],
               split_build_s=round(t_split, 1), evaluate_first_s=round(t_first, 3), evaluate_s=round(t_eval, 3),
               stages_s={k: round(v, 4) for k, v in timings.items()},
               kernel_ms={n.replace("sam6d_bop_", ""): round(kern[n], 3) for n in names}, kernel_calls=calls,
               evaluate_bbox_s=round(t_bbox, 3), AP=scores["AP"], AR100=scores["AR100"], AP_bbox=bb["AP"],
               oracle_s_per_image=round(t_oracle, 2), oracle_images=len(sub), oracle_arrays_equal=same)
    print(json.dumps(rec))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bop_coco_bench.json"), "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
