"""Time TSDF fusion and mesh extraction on the GPU (sam6d_b200/fusion.py, csrc/fusion.cu).

    python tools/fusion_bench.py [--out result.json]

300 views at 480 x 640 of a rendered closed mesh (tests/_symmetry_meshes "blob", 400 mm away, 642-view sphere) are fused
into 128^3, 256^3 and 384^3 volumes over the object's box, then the mesh is extracted from each.  Each stage is timed with
CUDA events after a warm-up run of the same shape.  Reported per size:
- integration: ms, voxel-view updates/s (voxels x views / time), and bytes/s against the bytes the rule must move: every
  voxel's 24 bytes read and written once per launch, plus each view's K and pose; the pixels a voxel reads are gathers
  that the rule does not bound, so they are left out (the figure is a floor on the traffic, not a roofline);
- extraction (count, both prefix sums, the totals' copy, emit): ms, and bytes/s against one read of tsdf and weight per pass
  (2 x 8 bytes per voxel), the mask and counts written and read, and the output written.
Prints the card's name, power limit and clocks, then one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from hypotheses_bench import card  # noqa: E402


def timed(fn, n=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--views", type=int, default=300)
    args = ap.parse_args()
    from sam6d_b200 import fusion, ops, render
    import _symmetry_meshes as sm
    assert torch.cuda.is_available(), "fusion_bench needs a GPU"
    H, W, f = 480, 640, 600.0
    mesh = sm.build("blob")
    poses = render.template_poses(level=2, distance=400.0)[:args.views]
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]])
    Kr = K.copy()
    Kr[:2, 2] += 0.5
    out = render.render([render.upload(mesh)], torch.from_numpy(poses.astype(np.float32))[None].cuda(), Kr, H, W, ambient=1.0)
    rgb, depth, mask = out["rgb"][0].contiguous(), out["depth"][0].contiguous(), out["mask"][0].contiguous()
    T = len(poses)
    K4, P12 = (torch.from_numpy(x).cuda() for x in fusion.pack_views(K, poses, T))
    res = dict(card=card(), views=T, height=H, width=W, sizes=[])
    print("[fusion_bench]", res["card"])
    for res_n in (128, 256, 384):
        lo, hi, voxel, trunc = fusion.view_bounds(depth, mask, K, poses, 1.0, resolution=res_n - 12)
        vol = fusion.TsdfVolume(lo, hi, voxel, trunc)
        N = vol.nx * vol.ny * vol.nz

        def integrate():
            vol.tsdf.fill_(1.0)
            vol.weight.zero_()
            vol.csum.zero_()
            vol.ccount.zero_()
            ops.tsdf_integrate(rgb, depth, mask, K4, P12, vol.tsdf, vol.weight, vol.csum, vol.ccount, vol.bbox_min,
                               float(np.float32(vol.voxel)), float(np.float32(vol.trunc)), fusion.ZNEAR_MM)

        def integrate_only():
            ops.tsdf_integrate(rgb, depth, mask, K4, P12, vol.tsdf, vol.weight, vol.csum, vol.ccount, vol.bbox_min,
                               float(np.float32(vol.voxel)), float(np.float32(vol.trunc)), fusion.ZNEAR_MM)

        integrate()
        t_int, _ = timed(integrate_only)            # the timed window is the kernel alone (its volume keeps accumulating)
        integrate()
        t_mesh, (v, c, fc) = timed(lambda: vol.mesh_tensors(1))
        ncube = (vol.nx - 1) * (vol.ny - 1) * (vol.nz - 1)
        int_bytes = N * 24 * 2 + T * 64
        mesh_bytes = N * 8 * 2 + N * 4 * 2 + N * 4 * 3 + ncube * 4 * 3 + len(v) * 15 + len(fc) * 12 + N * 16
        row = dict(dims=vol.dims, voxel_mm=vol.voxel, integrate_ms=t_int, updates_per_s=N * T / (t_int * 1e-3),
                   integrate_bytes_per_s=int_bytes / (t_int * 1e-3), mesh_ms=t_mesh, mesh_bytes_per_s=mesh_bytes / (t_mesh * 1e-3),
                   vertices=len(v), faces=len(fc))
        res["sizes"].append(row)
        print(f"[fusion_bench] {vol.dims}: integrate {t_int:.2f} ms ({row['updates_per_s'] / 1e9:.1f} G voxel-view updates/s, "
              f"{row['integrate_bytes_per_s'] / 1e9:.2f} GB/s floor traffic), mesh {t_mesh:.2f} ms "
              f"({row['mesh_bytes_per_s'] / 1e9:.1f} GB/s), {len(v)} vertices, {len(fc)} faces")
        del vol
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
