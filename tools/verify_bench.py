"""Time the pose verification (ops.verify_poses: render.render, then the count kernel of csrc/verify.cu) at P = 1 / 32 / 200
hypotheses of a 480 x 640 frame, and its share of a SAM6D.detect_objects frame, on the GPU.

    python tools/verify_bench.py [--P 1 32 200] [--reps 20] [--segmentor fastsam]

The scene is tests/test_gpu_verify.py's: the 1.6 k-face hull mesh (radius 110 mm) at 0.65 m with a second object hiding
about 30 % of it, 1 mm depth noise, K with f = 600; the hypotheses are the true pose perturbed by up to 20 degrees and 15 mm.
The render (in verify_poses' chunks) and the count kernel are timed separately with CUDA events around back-to-back calls;
the count is timed on the validated arguments (ops._pose_verify), so its window holds the memset, the launch and the
ctypes call.  The kernel's rate is the bytes it reads, 4 B of rendered depth and 1 B of mask per hypothesis pixel plus the
4 B per pixel observed depth once, over that time; every hypothesis here reads mask row 0, so the mask bytes come mostly from
L2 and the DRAM traffic is about 4 B per hypothesis pixel.  At small P the window is launch overhead, not bandwidth.
verify_poses is the host clock around whole calls.  The detect_objects frame
(seeded random weights: its proposal count, and so its time, is not that of trained weights) is the host clock over 5 frames
after 2 warm-up frames, without and with verify.  Prints the card's name and power limit, then one JSON line."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[1, 32, 200])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--segmentor", default="fastsam", choices=("fastsam", "sam"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import test_gpu_verify as tv
    from oracle import icp_oracle as io
    from sam6d_b200 import meshio, ops, render
    from sam6d_b200.pipeline import SAM6D
    print(f"[verify_bench] card: {card()}")
    meshes, ((R0, t0), _), depth, masks, hidden = tv._scene(1)
    H, W = depth.shape
    tau = 0.1 * tv._radius(meshes, 0)
    rows = []
    for P in args.P:
        rng = np.random.RandomState(P)
        R = np.stack([R0 @ io.so3_exp(np.radians(rng.uniform(0, 20)) * (a / np.linalg.norm(a))) for a in rng.normal(size=(P, 3))])
        t = t0 + rng.uniform(-0.015, 0.015, size=(P, 3))
        Rd, td = torch.from_numpy(R.astype(np.float32)).cuda(), torch.from_numpy(t.astype(np.float32)).cuda()
        poses = np.stack([tv._pose(r, x) for r, x in zip(R, t)])
        mrow = np.zeros(P, np.int64)
        step = max(1, ops.VERIFY_RENDER_BYTES // (26 * H * W))
        chunks = [torch.from_numpy(poses[i:i + step])[:, None].cuda() for i in range(0, P, step)]
        rdepth = tv._render_depth([meshes[0]] * P, poses)
        ms_render = events(lambda: [render.render([meshes[0]] * len(c), c, tv.K, H, W) for c in chunks], args.reps)
        mrow_h, tau_h = ops.verify_rows(mrow, tau, P, masks.shape[0])
        counts = torch.empty(P, 6, dtype=torch.int32, device="cuda")
        ms_count = events(lambda: ops._pose_verify(rdepth, depth, masks, mrow_h, tau_h, 1e-3, counts), args.reps)
        ms_verify = wall(lambda: ops.verify_poses(Rd, td, np.zeros(P, np.int64), meshes, depth, masks, mrow, tv.K, tau), args.reps, 2)
        nbytes = P * H * W * 5 + H * W * 4
        row = dict(P=P, render_ms=round(ms_render, 3), count_ms=round(ms_count, 4), count_GBps=round(nbytes / ms_count / 1e6, 1),
                   count_MB=round(nbytes / 1e6, 1), verify_poses_ms=round(ms_verify, 3))
        print(f"[verify_bench] P={P}: render {ms_render:.3f} ms, count {ms_count:.4f} ms ({row['count_GBps']} GB/s over "
              f"{row['count_MB']} MB), verify_poses {ms_verify:.3f} ms")
        rows.append(row)
        del rdepth
        torch.cuda.empty_cache()
    # a detect_objects frame of the same scene, without and with verification
    from test_gpu_icp import hull_mesh_mm
    v, f = hull_mesh_mm(os.path.join(ROOT, "tests", "golden"))
    cols = np.random.RandomState(0).randint(40, 255, (len(v), 3)).astype(np.uint8)
    mesh = meshio.Mesh(vertices=v, faces=f, colors=cols)
    sam6d = SAM6D(segmentor=args.segmentor, random_weights=True, verify=True)
    objs = sam6d.onboard_objects([mesh], template_size=256, rng=np.random.RandomState(0))
    raw = np.round(depth.cpu().numpy() * 1000.0).astype(np.uint16)
    rgb = np.full((H, W, 3), 90, np.uint8)
    rgb[raw > 0] = (200, 120, 40)
    frame = (rgb, raw, tv.K.ravel().tolist(), 1.0)
    detect = {}
    for on in (False, True):
        sam6d.verify = on
        detect[on] = wall(lambda: sam6d.detect_objects(*frame, objs, rng=np.random.RandomState(0)), 5, 2)
    n_pem = len(sam6d.detect_objects(*frame, objs, rng=np.random.RandomState(0)).pem)
    share = (detect[True] - detect[False]) / detect[True]
    print(f"[verify_bench] detect_objects frame ({args.segmentor}, {n_pem} poses): {detect[False]:.1f} ms without, "
          f"{detect[True]:.1f} ms with verify ({100 * share:.1f} %)")
    print(json.dumps(dict(card=card(), hidden=round(hidden, 3), rows=rows, detect_ms=round(detect[False], 2),
                          detect_verify_ms=round(detect[True], 2), detect_poses=n_pem, verify_share=round(share, 4))))


if __name__ == "__main__":
    main()
