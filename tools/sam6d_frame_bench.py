"""Times one whole SAM-6D frame (480 x 640, templates -> ISM -> PEM) through a resident sam6d_b200.pipeline.SAM6D and writes
one JSON file:
  * configurations: SAM ViT-H, SAM ViT-B, FastSAM-x and FastSAM-s as the segmentor, DINOv2 ViT-L descriptors, PEM in bf16; seeded weights
    (speed does not depend on their values);
  * frame: the repository's example frame (tests/golden/pem_input.pt) and the convex hull of its object's samples as the CAD;
  * per stage (segmentor, descriptors, scores, RLE, ISM records, PEM inputs, Net.forward, PEM records): host clock between
    device synchronisations, mean over --frames frames after --warmup frames; frames/s from a separate run of the same frames
    without the stage synchronisations;
  * the one-time onboard() cost (42 templates at 512 x 512, ISM references, PEM template bank), after one warm-up onboard;
  * the RLE hand-off: ops.mask_rle on the frame's proposal masks (CUDA events) against .cpu() + mask_to_rle per mask.
Thresholds: with seeded weights every score is arbitrary, so the counts are chosen.  The AMG keeps every mask its NMS keeps
(stability 0, predicted IoU -10, 32 x 32 points), FastSAM its max_det 200, the semantic threshold keeps all proposals (the
descriptor model runs on all of them in any case), and det_score_thresh is set between the --pem_dets-th and the next ISM
score so that --pem_dets detections reach the PEM.  The count after each filter is reported beside the times.
The card's name, power limit and SM clocks are read with nvidia-smi in the same run.  Without a CUDA device it fails.

With --objects 1,8,21 the first configuration instead times SAM6D.detect_objects on O onboarded objects for each O (the
example CAD at O distinct scales, ids 1..O): the stages above plus the per-object NMS ("nms"), onboard_objects' cost, and the
counts after each filter.

    python tools/sam6d_frame_bench.py [--frames 10] [--warmup 2] [--pem_dets 8] [--configs sam_vit_h,sam_vit_b,fastsam,fastsam_s]
                                      [--objects 1,8,21] --out FILE"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {
    "sam_vit_h": dict(segmentor="sam", sam_model_type="vit_h", stability_score_thresh=0.0, pred_iou_thresh=-10, points_per_side=32),
    "sam_vit_b": dict(segmentor="sam", sam_model_type="vit_b", stability_score_thresh=0.0, pred_iou_thresh=-10, points_per_side=32),
    "fastsam": dict(segmentor="fastsam"),
    "fastsam_s": dict(segmentor="fastsam", fastsam_model="FastSAM-s"),
}
STAGES = ("segmentor", "descriptors", "scores", "rle", "ism_records", "pem_inputs", "forward", "pem_records")
MULTI_STAGES = ("segmentor", "descriptors", "scores", "nms", "rle", "ism_records", "pem_inputs", "forward", "pem_records")


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                          check=True).stdout.strip().splitlines()[0]


def _example(tmp):
    """the example frame and its convex-hull CAD (PLY in mm)"""
    from scipy.spatial import ConvexHull
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "pem_input.pt"), weights_only=False)
    pts = gold["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    verts, faces = pts[hull.vertices], np.array([[remap[a] for a in s] for s in hull.simplices])
    cols = np.random.RandomState(0).randint(40, 255, (len(verts), 3))
    cad = os.path.join(tmp, "obj.ply")
    with open(cad, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                 % (len(verts), len(faces)))
        for v, c in zip(verts, cols):
            fh.write("%f %f %f %d %d %d\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
        for f in faces:
            fh.write("3 %d %d %d\n" % tuple(f))
    frame = (gold["rgb"].numpy().astype(np.uint8), gold["depth"].numpy().astype(np.uint16), gold["cam_K"], gold["depth_scale"])
    return cad, frame


class StageClock:
    """mark(stage): synchronise the device, add the host time since the previous mark to that stage"""

    def __init__(self, stages=STAGES):
        self.acc = {s: 0.0 for s in stages}
        self.t = None

    def start(self):
        torch.cuda.synchronize()
        self.t = time.perf_counter()

    def __call__(self, stage):
        torch.cuda.synchronize()
        now = time.perf_counter()
        self.acc[stage] += now - self.t
        self.t = now


def _rle_compare(masks, iters=20):
    from sam6d_b200 import ops
    from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle
    for _ in range(3):
        ops.mask_rle(masks)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.mask_rle(masks)
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / iters                     # includes the one 4-byte copy that sizes the output
    host = []
    for _ in range(3):
        torch.cuda.synchronize()
        t = time.perf_counter()
        m = masks.cpu().numpy()
        [mask_to_rle(m[i] > 0) for i in range(len(m))]
        host.append((time.perf_counter() - t) * 1e3)
    return dict(n_masks=int(masks.shape[0]), kernel_ms=round(kernel_ms, 3), host_copy_plus_numpy_ms=round(min(host), 2),
                mask_bytes=int(masks.numel() * 4))


def bench(name, cad, frame, args):
    from sam6d_b200.pipeline import SAM6D
    model = SAM6D(**CONFIGS[name], dinov2_model="dinov2_vitl14", precision="bf16", random_weights=True, confidence_thresh=-1,
                  det_score_thresh=-1)
    model.onboard(cad, template_size=512, rng=np.random.RandomState(0))      # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    obj = model.onboard(cad, template_size=512, rng=np.random.RandomState(0))
    torch.cuda.synchronize()
    onboard_ms = (time.perf_counter() - t) * 1e3
    # det_score_thresh between the pem_dets-th and the next ISM score
    res = model(*frame, obj, rng=np.random.RandomState(5))
    s = sorted((r["score"] for r in res.ism), reverse=True)
    if len(s) > args.pem_dets:
        model.det_score_thresh = 0.5 * (s[args.pem_dets - 1] + s[args.pem_dets])
    for _ in range(args.warmup):
        res = model(*frame, obj, rng=np.random.RandomState(5))
    clock = StageClock()
    for _ in range(args.frames):
        clock.start()
        res = model(*frame, obj, rng=np.random.RandomState(5), mark=clock)
    stages_ms = {k: round(v * 1e3 / args.frames, 2) for k, v in clock.acc.items()}
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(args.frames):
        model(*frame, obj, rng=np.random.RandomState(5))
    torch.cuda.synchronize()
    frame_ms = (time.perf_counter() - t) * 1e3 / args.frames
    counts = dict(proposals=res.n_proposals, semantic_kept=len(res.ism),
                  above_det_score_thresh=sum(r["score"] > model.det_score_thresh for r in res.ism), pem_kept=len(res.pem))
    out = dict(stages_ms=stages_ms, stage_sum_ms=round(sum(stages_ms.values()), 2), frame_ms=round(frame_ms, 2),
               frames_per_s=round(1e3 / frame_ms, 2), onboard_ms=round(onboard_ms, 1), counts=counts,
               det_score_thresh=model.det_score_thresh, rle=_rle_compare(res.masks.contiguous()))
    del model, obj, res
    torch.cuda.empty_cache()
    return out


def bench_objects(name, cad, frame, n_objects, args):
    """one detect_objects frame on n_objects objects: the example CAD scaled by 0.6 .. 1.4, ids 1..O"""
    from sam6d_b200 import meshio
    from sam6d_b200.pipeline import SAM6D
    model = SAM6D(**CONFIGS[name], dinov2_model="dinov2_vitl14", precision="bf16", random_weights=True, confidence_thresh=-1,
                  det_score_thresh=-1)
    base = meshio.load_ply_mesh(cad)
    scales = np.linspace(0.6, 1.4, n_objects) if n_objects > 1 else [1.0]
    meshes = [meshio.Mesh(vertices=(base.vertices * s).astype(np.float32), faces=base.faces, colors=base.colors) for s in scales]
    model.onboard_objects(meshes[:1], template_size=512, rng=np.random.RandomState(0))      # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    objs = model.onboard_objects(meshes, template_size=512, rng=np.random.RandomState(0))
    torch.cuda.synchronize()
    onboard_ms = (time.perf_counter() - t) * 1e3
    res = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    s = sorted((r["score"] for r in res.ism), reverse=True)
    if len(s) > args.pem_dets:
        model.det_score_thresh = 0.5 * (s[args.pem_dets - 1] + s[args.pem_dets])
    for _ in range(args.warmup):
        res = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    clock = StageClock(MULTI_STAGES)
    for _ in range(args.frames):
        clock.start()
        res = model.detect_objects(*frame, objs, rng=np.random.RandomState(5), mark=clock)
    stages_ms = {k: round(v * 1e3 / args.frames, 2) for k, v in clock.acc.items()}
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(args.frames):
        model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    torch.cuda.synchronize()
    frame_ms = (time.perf_counter() - t) * 1e3 / args.frames
    counts = dict(proposals=res.n_proposals, ism_after_nms=len(res.ism), objects_detected=len({r["category_id"] for r in res.ism}),
                  above_det_score_thresh=sum(r["score"] > model.det_score_thresh for r in res.ism), pem_kept=len(res.pem))
    out = dict(objects=n_objects, stages_ms=stages_ms, stage_sum_ms=round(sum(stages_ms.values()), 2), frame_ms=round(frame_ms, 2),
               frames_per_s=round(1e3 / frame_ms, 2), onboard_objects_ms=round(onboard_ms, 1), counts=counts,
               det_score_thresh=model.det_score_thresh, ref_patch_bytes=int(objs.ref_patch.numel() * objs.ref_patch.element_size()))
    del model, objs, res
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pem_dets", type=int, default=8, help="detections that reach the PEM (sets det_score_thresh)")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--objects", default=None, help="comma-separated object counts: time detect_objects instead (first config)")
    ap.add_argument("--out", required=True, help="JSON file to write")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sam6d_frame_bench needs a CUDA device")
    res = dict(card_before=_card(), frames=args.frames, warmup=args.warmup, pem_dets=args.pem_dets)
    with tempfile.TemporaryDirectory() as tmp:
        cad, frame = _example(tmp)
        if args.objects:
            name = args.configs.split(",")[0]
            for n in (int(x) for x in args.objects.split(",")):
                res[f"{name}_objects_{n}"] = bench_objects(name, cad, frame, n, args)
                print(name, json.dumps(res[f"{name}_objects_{n}"]), flush=True)
        else:
            for name in args.configs.split(","):
                res[name] = bench(name, cad, frame, args)
                print(name, json.dumps(res[name]), flush=True)
    res["card_after"] = _card()
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
