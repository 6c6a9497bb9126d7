"""Time BOP19 scoring on the GPU: the two kernels of csrc/bop_eval.cu (CUDA events, C entry points on preallocated inputs) and a
whole evaluate_bop19, against the float64 oracle (oracle/bop_eval_oracle.py) on the host cores, on a synthetic split.

    python tools/bop_eval_bench.py [--images 300] [--detail 16] [--oracle_pairs 40] [--out DIR]

The split (tests/test_gpu_bop_eval.py's builder): 640 x 480 images with 8 instances each (an ellipsoid, a cylinder with a
continuous symmetry about z, a box with a discrete one; two instances of most objects per image), meshes at models_eval-like
vertex counts, and two estimates per GT instance (tests/test_gpu_bop_eval.py: write_results "perturbed").  Prints the card's name and
power limit, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=300)
    ap.add_argument("--detail", type=int, default=16, help="mesh resolution (16: 10242 / 770 / 6534 vertices)")
    ap.add_argument("--oracle_pairs", type=int, default=40, help="pairs the float64 oracle scores on the host (timed per pair)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import test_gpu_bop_eval as tb
    from oracle import bop_eval_oracle as bo
    from oracle import render_oracle as ro
    from sam6d_b200 import _lib, bop_eval, meshio, render
    print(f"[bop_eval_bench] card: {card()}")

    work = tempfile.mkdtemp(prefix="bop_eval_bench_")
    rng = np.random.RandomState(0)
    objs = [1, 1, 2, 2, 3, 3, 1, 2]
    images = [(1 + i // 100, i % 100, 480, 640, 600.0, [(o, float(rng.uniform(0.05, 1.0))) for o in objs]) for i in range(args.images)]
    v1, f1 = ro.icosphere(5 if args.detail >= 16 else 3, 1.0)
    meshes = {1: (v1 * np.array([40.0, 25.0, 15.0], np.float32), f1), 2: tb.cylinder(20.0, 50.0, 24 * args.detail),
              3: tb.box(25.0, 15.0, 10.0, 2 * args.detail)}
    t0 = time.perf_counter()
    gts = tb.write_split(work, "synth", images, meshes)
    csv = tb.write_results(os.path.join(work, "result_synth.csv"), gts, "perturbed")
    t_split = time.perf_counter() - t0

    # whole evaluation: a first (cold) and a second run
    t0 = time.perf_counter()
    scores = bop_eval.evaluate_bop19(work, "synth", csv)
    torch.cuda.synchronize()
    t_first = time.perf_counter() - t0
    t0 = time.perf_counter()
    scores = bop_eval.evaluate_bop19(work, "synth", csv)
    torch.cuda.synchronize()
    t_eval = time.perf_counter() - t0
    P = scores["n_pairs"]

    # the kernels alone, on the split's own pairs
    res = bop_eval.load_results(csv)
    keys = {}
    for g in gts:
        keys.setdefault((g["scene_id"], g["im_id"], g["obj_id"]), []).append(g)
    pairs = [(r, g) for r in range(len(res["score"])) for g in keys.get((int(res["scene_id"][r]), int(res["im_id"][r]), int(res["obj_id"][r])), [])]
    info = bop_eval.load_models_info(os.path.join(work, "synth", "models_eval", "models_info.json"))
    syms = []
    for o in (1, 2, 3):
        R, t = bop_eval.symmetry_transforms(info[o])
        syms.append(torch.from_numpy(np.concatenate([R.reshape(-1, 9), t], 1).astype(np.float32)).cuda())
    dev = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)  # noqa: E731
    est = dev(np.array([np.r_[res["R"][r].reshape(-1), res["t"][r]] for r, _ in pairs]))
    gtp = dev(np.array([np.r_[g["R"].reshape(-1), g["t"]] for _, g in pairs]))
    pobj = dev(np.array([g["obj_id"] - 1 for _, g in pairs]), torch.int32)
    Kp = dev(np.tile([600.0, 600.0, 319.5, 240.25], (len(pairs), 1)))
    verts = [dev(meshes[o][0]) for o in (1, 2, 3)]
    V, S = torch.cat(verts).contiguous(), torch.cat(syms).contiguous()
    voff = dev(np.cumsum([0] + [len(meshes[o][0]) for o in (1, 2, 3)]), torch.int32)
    soff = dev(np.cumsum([0] + [len(s) for s in syms]), torch.int32)
    res_d = torch.empty(len(pairs), 2, dtype=torch.float32, device="cuda")
    ms_mssd = events(lambda: _lib.call("sam6d_bop_mssd_mspd", est, gtp, pobj, Kp, len(pairs), V, voff, S, soff, 3,
                                       max(len(s) for s in syms), res_d), 10)
    ref = bop_eval.mssd_mspd(est, gtp, pobj, Kp, verts, syms)
    assert torch.equal(ref, res_d)
    n_eval = sum(len(meshes[g["obj_id"]][0]) * len(syms[g["obj_id"] - 1]) for _, g in pairs)

    n_vsd = 256
    mesh = render.upload(meshio.Mesh(*meshes[1]))
    sel = [i for i, (_, g) in enumerate(pairs) if g["obj_id"] == 1][:n_vsd]
    poses = np.zeros((1, 2 * len(sel), 4, 4), np.float32)
    for k, i in enumerate(sel):
        r, g = pairs[i]
        poses[0, k, :3, :3], poses[0, k, :3, 3] = res["R"][r], res["t"][r]
        poses[0, len(sel) + k, :3, :3], poses[0, len(sel) + k, :3, 3] = g["R"], g["t"]
    poses[0, :, 3, 3] = 1
    K = np.array([[600.0, 0, 319.5], [0, 600.0, 240.25], [0, 0, 1]])
    depth = render.render([mesh], torch.from_numpy(poses).cuda(), K, 480, 640)["depth"][0]
    de, dg = depth[:len(sel)].contiguous(), depth[len(sel):].contiguous()
    dt = dg[:1].contiguous()
    img = torch.zeros(len(sel), dtype=torch.int32, device="cuda")
    taus = torch.from_numpy(bop_eval.VSD_TAUS.astype(np.float32)).cuda()
    out = torch.empty(len(sel), 12, dtype=torch.int32, device="cuda")
    ms_vsd = events(lambda: _lib.call("sam6d_bop_vsd_counts", de, dg, dt, img, len(sel), 480, 640, 600.0, 600.0, 319.5, 240.25, 15.0, 80.0,
                                      taus, out), 20)
    vsd_bytes = 2 * len(sel) * 480 * 640 * 4 + 480 * 640 * 4
    ms_render = events(lambda: render.render([mesh], torch.from_numpy(poses).cuda(), K, 480, 640), 3)

    # the oracle on the host, per pair: MSSD + MSPD over the symmetry set, VSD counts from the same depth images
    no = min(args.oracle_pairs, len(pairs))
    osel = list(range(0, len(pairs), max(1, len(pairs) // no)))[:no]
    t0 = time.perf_counter()
    for i in osel:
        r, g = pairs[i]
        X = meshes[g["obj_id"]][0].astype(np.float64)
        s = bo.symmetries(info[g["obj_id"]])
        bo.mssd(res["R"][r], res["t"][r], g["R"], g["t"], X, s)
        bo.mspd(res["R"][r], res["t"][r], g["R"], g["t"], X, s, K)
    t_or_ms = (time.perf_counter() - t0) / len(osel)
    dcpu = [(de[k].cpu().numpy(), dg[k].cpu().numpy()) for k in range(min(no, len(sel)))]
    dtc = dt[0].cpu().numpy()
    t0 = time.perf_counter()
    for a, b in dcpu:
        bo.vsd_counts(a, b, dtc, K, 15.0, 80.0)
    t_or_vsd = (time.perf_counter() - t0) / len(dcpu)
    n_cont = sum(g["obj_id"] == 2 for _, g in pairs)
    rec = dict(card=card(), images=args.images, pairs=P, pairs_continuous_symmetry=int(n_cont),
               vertices={o: int(len(meshes[o][0])) for o in meshes}, symmetries={o: int(len(syms[o - 1])) for o in (1, 2, 3)},
               split_build_s=round(t_split, 2), evaluate_first_s=round(t_first, 3), evaluate_s=round(t_eval, 3),
               ar=scores["ar"], mssd_mspd_kernel_ms=round(ms_mssd, 3), mssd_mspd_vertex_symmetry_evals_per_s=float(f"{n_eval / ms_mssd * 1e3:.3e}"),
               vsd_kernel_ms_256_pairs=round(ms_vsd, 4), vsd_kernel_gbs=round(vsd_bytes / ms_vsd / 1e6, 1),
               render_ms_512_views=round(ms_render, 3), oracle_mssd_mspd_ms_per_pair=round(t_or_ms * 1e3, 2),
               oracle_vsd_counts_ms_per_pair=round(t_or_vsd * 1e3, 2), oracle_pairs_timed=len(osel))
    print(json.dumps(rec))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bop_eval_bench.json"), "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
