"""tools/render_bench.py -- times the template rasteriser (sam6d_b200.render.render) on procedural meshes and prints one JSON line.

Cases, all at 512 x 512 with the 42 level-0 views (render_custom_templates framing, d = 4 r):
    ico80k    one icosphere of 81 920 triangles (a typical scanned CAD model)
    ico1m     one icosphere of 1 310 720 triangles
    ycbv21    21 objects x 42 views in one call (YCB-V-shaped: 21 icospheres of 20 480 triangles, different radii and colours)
    splat80k  the CPU point-splat stand-in (cli/render_point_templates.py, 400 k samples) on the ico80k mesh, for context
GPU times are CUDA events around render() (host packing included) on the current stream, median of --reps after --warmup calls;
the card's name, power limit and SM clock are read in the same run.

Usage: python tools/render_bench.py [--reps 10 --warmup 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import render_oracle as ro  # noqa: E402
from sam6d_b200 import meshio, render  # noqa: E402
from sam6d_b200.cli import render_point_templates as rpt  # noqa: E402

SIZE = 512


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(["gpu", "power_limit", "sm_clock", "sm_clock_max"], vals))
    except Exception as e:                                      # report, do not guess
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def _time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts))


def _case(meshes_np, radii, reps, warmup):
    meshes = [render.upload(m) for m in meshes_np]
    poses = torch.from_numpy(np.stack([render.level0_template_poses(4.0 * r) for r in radii]).astype(np.float32)).cuda()
    K = render.template_K(SIZE)
    out = render.render(meshes, poses, K, SIZE, SIZE)
    torch.cuda.synchronize()
    med, best = _time(lambda: render.render(meshes, poses, K, SIZE, SIZE), reps, warmup)
    views = poses.shape[0] * poses.shape[1]
    return dict(ms=round(med, 3), ms_min=round(best, 3), views=views, views_per_s=round(views / (med / 1e3), 1),
                triangles=int(sum(m.faces.shape[0] for m in meshes_np)), dropped=int(out["dropped"].sum()),
                covered_px=int((out["mask"] > 0).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "render_bench needs a GPU"
    rng = np.random.RandomState(0)
    res = {"bench": "render", "size": SIZE}
    res.update(_gpu_info())

    v, f = ro.icosphere(6, 50.0)
    col = rng.randint(0, 256, (len(v), 3)).astype(np.uint8)
    ico80k = meshio.Mesh(v, f, col)
    res["ico80k"] = _case([ico80k], [50.0], a.reps, a.warmup)

    v1, f1 = ro.icosphere(8, 50.0)
    res["ico1m"] = _case([meshio.Mesh(v1, f1)], [50.0], a.reps, a.warmup)

    v5, f5 = ro.icosphere(5, 1.0)
    radii = rng.uniform(30.0, 120.0, 21)
    objs = [meshio.Mesh((v5 * r).astype(np.float32), f5, rng.randint(0, 256, (len(v5), 3)).astype(np.uint8)) for r in radii]
    res["ycbv21"] = _case(objs, list(radii), a.reps, a.warmup)

    t0 = time.perf_counter()
    rpt.render_templates(v, f.astype(np.int64), col, size=SIZE)
    res["splat80k_cpu"] = dict(ms=round((time.perf_counter() - t0) * 1e3, 1), views=42)
    after = _gpu_info()
    res["sm_clock_after"] = after.get("sm_clock")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
