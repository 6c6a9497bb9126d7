"""A small BOP test split with visible and full masks, and ISM-style detection JSONs for it, for the COCO scoring tests
(tests/test_bop_coco_cpu.py, tests/test_gpu_bop_coco.py) and tools/bop_coco_bench.py.

Masks are procedural ellipses and boxes that overlap; the full mask of an instance is its visible mask plus an occluded part.
Detections are uncompressed COCO RLEs (mask_to_rle, the ISM's writer) of perturbed GT masks plus false positives."""
import json
import os

import numpy as np

from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle

# (scene_id, im_id, H, W, [(obj_id, visib_fract, kind), ...]); kind: "" normal, "corner" touches pixel (0,0), "last" covers
# the last pixel, "big" covers most of the image (a large area), "empty" has an empty visible mask, "nofull" a visible mask but
# an empty full mask
IMAGES = [(1, 0, 96, 128, [(1, 0.9, "corner"), (2, 0.6, ""), (1, 0.099, ""), (3, 0.1, "last"), (2, 0.5, "empty")]),
          (1, 3, 96, 128, [(3, 0.11, "big"), (1, 0.05, ""), (2, 0.95, ""), (3, 0.7, "nofull"), (1, 0.8, "")]),
          (2, 1, 30, 41, [(2, 0.9, "corner"), (1, 0.3, "last"), (2, 0.12, ""), (3, 0.08, "")])]


def ellipse(H, W, cy, cx, ry, rx):
    y, x = np.mgrid[:H, :W]
    return ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 <= 1.0


def write_split(root, dataset="toy", images=IMAGES, seed=0):
    """root/dataset/test/<scene>/{rgb, mask, mask_visib, scene_gt.json, scene_gt_info.json, scene_camera.json} and
    test_targets_bop19.json -> {(scene_id, im_id): [(obj_id, visible mask (H,W) bool, full mask, visib_fract)]}"""
    from PIL import Image
    rng = np.random.RandomState(seed)
    ds = os.path.join(root, dataset)
    out, scenes, targets = {}, {}, []
    for s, im, H, W, insts in images:
        sdir = os.path.join(ds, "test", f"{s:06d}")
        for sub in ("rgb", "mask", "mask_visib"):
            os.makedirs(os.path.join(sdir, sub), exist_ok=True)
        Image.fromarray(np.zeros((H, W, 3), np.uint8)).save(os.path.join(sdir, "rgb", f"{im:06d}.png"))
        gt, info, cam = scenes.setdefault(s, ({}, {}, {}))
        gt[str(im)], info[str(im)] = [], []
        cam[str(im)] = {"cam_K": [500.0, 0, W / 2, 0, 500.0, H / 2, 0, 0, 1], "depth_scale": 1.0}
        occl = np.zeros((H, W), bool)
        recs, counts = [], {}
        for k, (o, vis, kind) in enumerate(insts):
            cy, cx = rng.uniform(0.2, 0.8) * H, rng.uniform(0.15, 0.85) * W
            ry, rx = rng.uniform(0.12, 0.45) * H, rng.uniform(0.1, 0.4) * W
            full = ellipse(H, W, cy, cx, ry, rx) if k % 2 == 0 else np.zeros((H, W), bool)
            if k % 2:
                y0, x0 = int(cy - ry), int(cx - rx)
                full[max(0, y0):int(cy + ry), max(0, x0):int(cx + rx)] = True
            if kind == "big":
                full[4:-4, 4:-4] = True
            if kind == "corner":
                full[:max(2, H // 5), :max(2, W // 6)] = True
            if kind == "last":
                full[H - max(2, H // 6):, W - max(2, W // 5):] = True
            visible = full & ~occl
            occl |= full & (rng.rand(H, W) < 0.7)
            if kind == "empty":
                visible[:] = False
            if kind == "nofull":
                full = np.zeros((H, W), bool)
                visible = ellipse(H, W, cy, cx, ry / 2, rx / 2)
            # stored values: any value > 0 is set
            val = rng.randint(1, 256, size=(H, W)).astype(np.uint8)
            Image.fromarray(np.where(visible, val, 0).astype(np.uint8)).save(os.path.join(sdir, "mask_visib", f"{im:06d}_{k:06d}.png"))
            Image.fromarray(np.where(full, 255, 0).astype(np.uint8)).save(os.path.join(sdir, "mask", f"{im:06d}_{k:06d}.png"))
            gt[str(im)].append({"cam_R_m2c": [1, 0, 0, 0, 1, 0, 0, 0, 1], "cam_t_m2c": [0, 0, 500], "obj_id": o})
            info[str(im)].append({"visib_fract": vis})
            recs.append((o, visible, full, vis))
            counts[o] = counts.get(o, 0) + 1
        out[(s, im)] = recs
        targets += [{"scene_id": s, "im_id": im, "obj_id": o, "inst_count": n} for o, n in counts.items()]
    # an image that is not a target
    s, im, H, W = 1, 7, 96, 128
    sdir = os.path.join(ds, "test", f"{s:06d}")
    Image.fromarray(np.zeros((H, W, 3), np.uint8)).save(os.path.join(sdir, "rgb", f"{im:06d}.png"))
    scenes[s][0][str(im)], scenes[s][1][str(im)] = [], []
    scenes[s][2][str(im)] = {"cam_K": [500.0, 0, W / 2, 0, 500.0, H / 2, 0, 0, 1], "depth_scale": 1.0}
    for s, (gt, info, cam) in scenes.items():
        sdir = os.path.join(ds, "test", f"{s:06d}")
        for name, obj in (("scene_gt", gt), ("scene_gt_info", info), ("scene_camera", cam)):
            with open(os.path.join(sdir, f"{name}.json"), "w") as fh:
                json.dump(obj, fh)
    with open(os.path.join(ds, "test_targets_bop19.json"), "w") as fh:
        json.dump(targets, fh)
    return out


def box_xywh(mask):
    ys, xs = np.nonzero(mask)
    if not len(xs):
        return [0, 0, 0, 0]
    return [int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1)]


def record(s, im, o, score, mask, bbox=None):
    return {"scene_id": s, "image_id": im, "category_id": o, "score": score, "bbox": bbox if bbox is not None else box_xywh(mask),
            "time": 0.5, "segmentation": mask_to_rle(mask.astype(np.uint8))}


def perturbed_detections(split, seed=1):
    """per GT instance one to three detections of shifted, dilated, eroded or noisy copies of its visible (or full) mask, with
    scores on a coarse grid (ties), float boxes with noise; false positives; a detection of an object and of an image that are
    not in the split"""
    rng = np.random.RandomState(seed)
    recs = []
    for (s, im), insts in split.items():
        H, W = insts[0][1].shape
        for o, vis, full, _ in insts:
            base = vis if vis.any() else full
            for j in range(rng.randint(1, 4)):
                m = np.roll(base, (rng.randint(-3, 4), rng.randint(-3, 4)), axis=(0, 1))
                if rng.rand() < 0.3:
                    m = m & (rng.rand(H, W) < 0.8)
                if rng.rand() < 0.3:
                    m = m | np.roll(m, 1, axis=0) | np.roll(m, 1, axis=1)
                bb = [float(v) + float(rng.uniform(-2, 2)) for v in box_xywh(m)]
                bb[2], bb[3] = max(bb[2], 0.5), max(bb[3], 0.5)
                recs.append(record(s, im, o, round(float(rng.uniform(0.1, 1.0)), 1), m, bb))
        for _ in range(3):
            m = ellipse(H, W, rng.uniform(0, H), rng.uniform(0, W), rng.uniform(2, H / 3), rng.uniform(2, W / 3))
            recs.append(record(s, im, int(rng.choice([1, 2, 3])), round(float(rng.uniform(0.1, 1.0)), 1), m))
        recs.append(record(s, im, 9, 0.99, insts[0][1]))
        recs.append(record(s, im, 1, 0.5, np.zeros((H, W), bool)))          # an empty mask
    recs.append(record(1, 7, 1, 0.99, np.ones((96, 128), bool)))
    order = rng.permutation(len(recs))
    return [recs[i] for i in order]


def write_json(path, recs):
    with open(path, "w") as fh:
        json.dump(recs, fh)
    return str(path)
