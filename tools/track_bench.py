"""Time a tracked frame (sam6d_b200/track.py: Tracker) at O = 1 / 8 / 21 objects, split into its render, point selection
(csrc/track.cu) and ICP (csrc/icp.cu), beside a SAM6D.detect_objects frame of the same objects, on the GPU.

    python tools/track_bench.py [--objects 1 8 21] [--reps 50] [--segmentor fastsam] [--max_instances 1]

The scene is tests/test_gpu_track.py's: a 480 x 640 frame, K with f = 600, the 1.6 k-face hull mesh (radius 110 mm) as every
object, O copies spread over the frame at 0.6 - 0.9 m with 1 mm depth noise.  Each object is seeded at its true pose, so every
track stays live (the loss rule is switched off here, so overlapping copies never trigger a detection).  The stages are timed with CUDA events around back-to-back calls at the tracker's shapes (N = 2048 points,
M = 4096 ICP samples, 10 ICP iterations); the tracked frame is the host clock around Tracker.__call__ (the render, the
selection, the ICP, the loss rule's device-to-host copy and the records), averaged over --reps frames after a warm-up.  The
detect_objects frame (FastSAM-x or SAM ViT-H and DINOv2 ViT-L with seeded random weights: its proposal count, and so its
time, is not that of trained weights) is the host clock over 5 frames after 2 warm-up frames.  Prints the card's name and
power limit, then one JSON line.

With --max_instances I > 1 every object is placed I times (L = O x I tracks, each copy seeded at its true pose), the tracker
runs with max_instances I, and point selection is timed both ways at the same L: the shared rule (ops.track_points) and the
exclusive one the tracker uses (ops.track_points_scene).  The detect_objects frame is not timed then."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def events(fn, n):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def wall(fn, n, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return 1000.0 * (time.perf_counter() - t0) / n


def scene(O, up, rng):
    """O poses spread over the frame and the frame's raw depth"""
    import test_gpu_track as tt
    poses = []
    for o in range(O):
        z = 0.6 + 0.3 * rng.rand()
        u, v = rng.uniform(120, 520), rng.uniform(100, 380)
        t = np.array([(u - tt.K[0, 2]) * z / tt.K[0, 0], (v - tt.K[1, 2]) * z / tt.K[1, 1], z])
        poses.append((tt._so3(rng.normal(size=3), rng.uniform(0, 180)), t))
    raw = tt.raw_depth(tt.render_depth_mm([up] * O, poses), rng)
    return poses, raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, nargs="+", default=[1, 8, 21])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--segmentor", default="fastsam", choices=("fastsam", "sam"))
    ap.add_argument("--max_instances", type=int, default=1, help="copies of each object, and tracks per object")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import test_gpu_track as tt
    from sam6d_b200 import meshio, ops, render
    from sam6d_b200.pipeline import SAM6D
    from sam6d_b200.track import Tracker
    print(f"[track_bench] card: {card()}")
    golden = os.path.join(ROOT, "tests", "golden")
    main_mesh, _, up = tt._meshes(golden)
    cols = np.random.RandomState(0).randint(40, 255, (len(main_mesh.vertices), 3)).astype(np.uint8)
    mesh = meshio.Mesh(vertices=main_mesh.vertices, faces=main_mesh.faces.astype(np.int64), colors=cols)
    sam6d = SAM6D(segmentor=args.segmentor, random_weights=True)
    rgb_bg = np.full((tt.H, tt.W, 3), 90, np.uint8)
    rows = []
    I = args.max_instances
    for O in args.objects:
        rng = np.random.RandomState(O)
        L = O * I
        poses, raw = scene(L, up[0], rng)
        rgb = rgb_bg.copy()
        rgb[raw > 0] = (200, 120, 40)
        objs = sam6d.onboard_objects([mesh] * O, template_size=256, rng=np.random.RandomState(0))
        # no loss and no re-detection: every timed frame is a tracked frame of all L tracks (the first call detects)
        tr = Tracker(sam6d, objs, [mesh] * O, redetect_interval=10 ** 9, min_inlier_fraction=0.0, max_rms_m=float("inf"),
                     max_instances=I, assoc_scale=0.0)
        for i, (R, t) in enumerate(poses):
            tr.start(i // I, R, t)
        tr(rgb, raw, tt.K.ravel(), tt.DEPTH_SCALE)
        live = tr.live.sum()
        # the stages at the tracker's shapes, from the tracker's own state
        R, t = tr.R.contiguous(), tr.t.contiguous()
        P = torch.zeros(L, 1, 4, 4, device="cuda")
        P[:, 0, :3, :3], P[:, 0, :3, 3], P[:, 0, 3, 3] = R, t * 1000.0, 1.0
        meshes = [tr.meshes[o] for o in tr.obj]
        rd = render.render(meshes, P, tt.K, tt.H, tt.W)["depth"][:, 0].contiguous()
        depth_d = torch.from_numpy(raw).cuda()
        obj = torch.from_numpy(tr.obj).cuda()
        centre = (torch.einsum("lij,lj->li", R, tr.centroid[obj]) + t).contiguous()
        gate = tr.gate_radius[obj].contiguous()
        pts, _, _ = ops.track_points(rd, depth_d, tt.DEPTH_SCALE, tt.K, centre, gate, tr.margin_px, tr.n_points)
        icp_radius, obj = tr.icp_radius[obj].contiguous(), obj.to(torch.int32)
        ms_render = events(lambda: render.render(meshes, P, tt.K, tt.H, tt.W), args.reps)
        ms_select = events(lambda: ops.track_points(rd, depth_d, tt.DEPTH_SCALE, tt.K, centre, gate, tr.margin_px, tr.n_points),
                           args.reps)
        ms_icp = events(lambda: ops.icp_refine(R, t, pts, tr.icp[0], tr.icp[1], obj, icp_radius, tr.track_icp_iters),
                        args.reps)
        ms_frame = wall(lambda: tr(rgb, raw, tt.K.ravel(), tt.DEPTH_SCALE), args.reps, 3)
        states = tr(rgb, raw, tt.K.ravel(), tt.DEPTH_SCALE).state
        if I == 1:
            ms_detect = wall(lambda: sam6d.detect_objects(rgb, raw, tt.K.ravel(), tt.DEPTH_SCALE, objs), 5, 2)
            row = dict(objects=O, live_after=int(live), tracked=states.count("tracked"), render_ms=round(ms_render, 3),
                       select_ms=round(ms_select, 3), icp_ms=round(ms_icp, 3), tracked_frame_ms=round(ms_frame, 3),
                       detect_frame_ms=round(ms_detect, 2), detect_over_tracked=round(ms_detect / ms_frame, 1))
            print(f"[track_bench] O={O}: render {ms_render:.3f} ms, select {ms_select:.3f} ms, ICP {ms_icp:.3f} ms; tracked frame "
                  f"{ms_frame:.3f} ms ({row['tracked']} of {O} tracked), detect_objects frame ({args.segmentor}) {ms_detect:.1f} ms")
        else:
            ms_scene = events(lambda: ops.track_points_scene(rd, depth_d, tt.DEPTH_SCALE, tt.K, centre, gate, tr.margin_px,
                                                             tr.n_points), args.reps)
            row = dict(objects=O, instances=I, tracks=L, live_after=int(live), tracked=states.count("tracked"),
                       render_ms=round(ms_render, 3), select_shared_ms=round(ms_select, 3), select_scene_ms=round(ms_scene, 3),
                       icp_ms=round(ms_icp, 3), tracked_frame_ms=round(ms_frame, 3))
            print(f"[track_bench] O={O} x {I} (L={L}): render {ms_render:.3f} ms, select track_points {ms_select:.3f} ms, "
                  f"track_points_scene {ms_scene:.3f} ms, ICP {ms_icp:.3f} ms; tracked frame {ms_frame:.3f} ms "
                  f"({row['tracked']} of {L} tracked)")
        rows.append(row)
        del tr, objs
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card(), segmentor=args.segmentor, rows=rows)))


if __name__ == "__main__":
    main()
