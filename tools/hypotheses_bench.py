"""Time several coarse hypotheses per proposal (Net.set_hypotheses) on the GPU.

    python tools/hypotheses_bench.py [--B 1 32 200] [--K 1 2 4 8] [--reps 10] [--out result.json]

- bf16 Net.forward replayed as a CUDA graph (the bench path: seeded synth weights and inputs, caller-provided uniforms) at every
  B x K, CUDA events around `reps` back-to-back calls after the sighting and the capture, with the peak device memory of the
  call (torch.cuda.max_memory_allocated after a reset, the inputs included).
- The coarse / fine split at B = 32: one fine pass is T(K = 2) - T(K = 1) of the replayed forward (it also holds the pick
  kernel, timed separately), the rest of T(K = 1) is the features, the geometric embedding and the coarse stage.
- The pick kernel alone (ops.coarse_pick_distinct on the arrays of a real forward, 30 degrees / 0.2 radii), CUDA events around
  200 launches.
- ops.verify_poses at P = B K on the rendered scene of tests/test_gpu_verify.py (host clock around whole calls).
- One SAM6D.detect_objects frame (FastSAM, seeded random weights: its proposal count is not that of trained weights) at K = 1
  and K = 4 with verify on, host clock over 5 frames after 2 warm-up frames.
Prints the card's name, power limit and maximum SM clock, then one JSON line."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
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
    ap.add_argument("--B", type=int, nargs="+", default=[1, 32, 200])
    ap.add_argument("--K", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from sam6d_b200 import ops, synth
    from sam6d_b200.pem import Net
    dev = torch.device("cuda")
    print(f"[hypotheses_bench] card: {card()}")
    net = Net(precision="bf16").to(dev).eval()
    net.load_state_dict(synth.make_pem_state_dict(seed=1), strict=True)
    keys = ("pts", "dense_fm", "dense_po", "dense_fo", "model")
    result = dict(card=card(), forward=[], pick=[], verify=[])
    T = {}
    for B in args.B:
        inp = {k: v.to(dev) for k, v in synth.make_pem_inputs(B=B, n=2048, n_model=1024, seed=100).items() if k in keys}
        rand = torch.rand(B, synth.N_PROPOSAL1 * 3, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        for K in args.K:
            net.set_hypotheses(K).enable_graphs()
            net(dict(inp), rand=rand)                                   # sighting (launch by launch)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            net(dict(inp), rand=rand)                                   # capture + replay
            ms = events(lambda: net(dict(inp), rand=rand), args.reps)
            peak = torch.cuda.max_memory_allocated() / 2 ** 20
            assert net._graphs.replays >= args.reps + 2
            T[B, K] = ms
            row = dict(B=B, K=K, ms=round(ms, 3), per_proposal_ms=round(ms / B, 4), peak_MiB=round(peak, 1))
            print(f"[hypotheses_bench] forward B={B} K={K}: {ms:.3f} ms ({ms / B:.4f} ms per proposal), peak {peak:.0f} MiB")
            result["forward"].append(row)
            net.disable_graphs()
            torch.cuda.empty_cache()
        # the pick kernel alone, on the arrays of a real forward
        rec = {}
        orig = ops.coarse_select

        def spy(*a):
            out = orig(*a)
            rec.update(Rt=a[0], top=a[1], scores=out[2])
            return out

        ops.coarse_select = spy
        net.set_hypotheses(1)(dict(inp), rand=rand)
        ops.coarse_select = orig
        for K in (4, 8):
            ms = events(lambda: ops.coarse_pick_distinct(rec["Rt"], rec["top"], rec["scores"], K, 30.0, 0.2), 200)
            cnt = ops.coarse_pick_distinct(rec["Rt"], rec["top"], rec["scores"], K, 30.0, 0.2)[4].float().mean().item()
            print(f"[hypotheses_bench] pick kernel B={B} K={K}: {1000 * ms:.1f} us, {cnt:.2f} distinct per proposal")
            result["pick"].append(dict(B=B, K=K, us=round(1000 * ms, 2), mean_count=round(cnt, 3)))
        del inp, rec
        torch.cuda.empty_cache()
    if (32, 1) in T and (32, 2) in T:
        fine = T[32, 2] - T[32, 1]
        result["split_B32"] = dict(step_ms=round(T[32, 1], 3), fine_pass_ms=round(fine, 3), rest_ms=round(T[32, 1] - fine, 3),
                                   fine_share=round(fine / T[32, 1], 4))
        print(f"[hypotheses_bench] B=32: step {T[32, 1]:.3f} ms, one fine pass {fine:.3f} ms ({100 * fine / T[32, 1]:.1f} %), "
              f"features + coarse stage {T[32, 1] - fine:.3f} ms")
    del net
    torch.cuda.empty_cache()
    # verification of all B K poses
    import test_gpu_verify as tv
    from oracle import icp_oracle as io
    meshes, ((R0, t0), _), depth, masks, hidden = tv._scene(1)
    tau = 0.1 * tv._radius(meshes, 0)
    for P in sorted({B * K for B in args.B for K in args.K}):
        rng = np.random.RandomState(P)
        R = np.stack([R0 @ io.so3_exp(np.radians(rng.uniform(0, 20)) * (a / np.linalg.norm(a))) for a in rng.normal(size=(P, 3))])
        t = t0 + rng.uniform(-0.015, 0.015, size=(P, 3))
        Rd, td = torch.from_numpy(R.astype(np.float32)).cuda(), torch.from_numpy(t.astype(np.float32)).cuda()
        ms = wall(lambda: ops.verify_poses(Rd, td, np.zeros(P, np.int64), meshes, depth, masks, np.zeros(P, np.int64), tv.K, tau),
                  3, 1)
        print(f"[hypotheses_bench] verify_poses P={P}: {ms:.3f} ms")
        result["verify"].append(dict(P=P, ms=round(ms, 3)))
    # a detect_objects frame with verification, one hypothesis against four
    from sam6d_b200 import meshio
    from sam6d_b200.pipeline import SAM6D
    from test_gpu_icp import hull_mesh_mm
    v, f = hull_mesh_mm(os.path.join(ROOT, "tests", "golden"))
    cols = np.random.RandomState(0).randint(40, 255, (len(v), 3)).astype(np.uint8)
    sam6d = SAM6D(segmentor="fastsam", random_weights=True, verify=True)
    objs = sam6d.onboard_objects([meshio.Mesh(vertices=v, faces=f, colors=cols)], template_size=256, rng=np.random.RandomState(0))
    H, W = depth.shape
    raw = np.round(depth.cpu().numpy() * 1000.0).astype(np.uint16)
    rgb = np.full((H, W, 3), 90, np.uint8)
    rgb[raw > 0] = (200, 120, 40)
    frame = (rgb, raw, tv.K.ravel().tolist(), 1.0)
    detect = {}
    for K in (1, 4):
        sam6d.pem.set_hypotheses(K)
        detect[K] = wall(lambda: sam6d.detect_objects(*frame, objs, rng=np.random.RandomState(0)), 5, 2)
    n_pem = len(sam6d.detect_objects(*frame, objs, rng=np.random.RandomState(0)).pem)
    print(f"[hypotheses_bench] detect_objects frame with verify ({n_pem} poses): {detect[1]:.1f} ms at K = 1, {detect[4]:.1f} ms at K = 4")
    result.update(detect_ms_K1=round(detect[1], 2), detect_ms_K4=round(detect[4], 2), detect_poses=n_pem)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
