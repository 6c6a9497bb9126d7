"""tools/ism_score_bench.py -- GPU (H100).  Times ISM template scoring and onboarding at each template level.

Scoring: sam6d_template_score_agg (csrc/ism.cu, the call behind ops.template_score) on preallocated outputs at P = 200 proposals, C = 1024 (DINOv2 ViT-L), O in {1, 21}, T in {42, 642}, every
aggregation, CUDA events around --iters launches after --warmup.  Reported with the reference bytes each launch reads
(ceil(P / 8) x O x T x C x 4: one pass over the references per tile of 8 proposals) and their share of the H100 SXM's
3.35 TB/s HBM3 (data sheet); repeated passes may hit L2, so this is a traffic figure, not a measured DRAM rate.
--baseline-lib times another build of libsam6d_b200.so (e.g. the previous kernel) through its sam6d_template_score entry
point (avg_5) on the same inputs, alternating with the current one; its reads are counted as P x O x T x C x 4 (one pass
per proposal, the one-CTA-per-proposal kernel).

Onboarding (--onboard): SAM6D(segmentor="fastsam", random_weights=True).onboard of a 1.6 k-face mesh at 512 x 512 for
level_templates 0 / 1 / 2 ("all") and 2 ("upper"): wall time (synchronised) and peak allocated device memory.

Prints the card's name and power limit first; writes JSON to --out.

Usage: python tools/ism_score_bench.py [--baseline-lib path/to/libsam6d_b200.so] [--onboard] [--out result.json]"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sam6d_b200 import _lib, ops  # noqa: E402
from sam6d_b200.synth import make_descriptors  # noqa: E402

HBM_BPS = 3.35e12
P, C, TILE = 200, 1024, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q)


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def scoring(args):
    base = None
    if args.baseline_lib:
        base = ctypes.CDLL(args.baseline_lib)
        base.sam6d_template_score.restype = ctypes.c_int
        base.sam6d_template_score.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 6
    rows = []
    for O in (1, 21):
        for T in (42, 642):
            q, r = make_descriptors(P=P, O=O, T=T, C=C, seed=O + T)
            qn, rn = ops.l2norm_rows(q.cuda()), ops.l2norm_rows(r.cuda())
            ref_bytes = O * T * C * 4
            obj, obj_t = torch.empty(P, O, device="cuda"), torch.empty(P, O, dtype=torch.int32, device="cuda")
            bo, bt = torch.empty(P, dtype=torch.int32, device="cuda"), torch.empty(P, dtype=torch.int32, device="cuda")
            bs = torch.empty(P, device="cuda")
            for agg, code in ops.TEMPLATE_AGGREGATIONS.items():
                def run():          # the C entry point on preallocated outputs, as the baseline below: kernel time, not Python
                    assert _lib.lib().sam6d_template_score_agg(qn.data_ptr(), rn.data_ptr(), P, O, T, C, code, None, obj.data_ptr(),
                                                               obj_t.data_ptr(), bo.data_ptr(), bs.data_ptr(), bt.data_ptr(),
                                                               torch.cuda.current_stream().cuda_stream) == 0
                ms = [time_ms(run, args.iters, args.warmup)]
                rec = dict(P=P, O=O, T=T, C=C, aggregation=agg, reads_bytes=math.ceil(P / TILE) * ref_bytes)
                if base is not None and agg == "avg_5":

                    def run_base():
                        rc = base.sam6d_template_score(qn.data_ptr(), rn.data_ptr(), P, O, T, C, None, obj.data_ptr(), bo.data_ptr(),
                                                       bs.data_ptr(), bt.data_ptr(), torch.cuda.current_stream().cuda_stream)
                        assert rc == 0, rc
                    bms = []
                    for _ in range(args.rounds):                        # alternate the two builds
                        bms.append(time_ms(run_base, args.iters, args.warmup))
                        ms.append(time_ms(run, args.iters, args.warmup))
                    rec.update(baseline_ms=float(np.median(bms)), baseline_reads_bytes=P * ref_bytes)
                    rec["baseline_hbm_share"] = rec["baseline_reads_bytes"] / (rec["baseline_ms"] * 1e-3) / HBM_BPS
                rec["ms"] = float(np.median(ms))
                rec["hbm_share"] = rec["reads_bytes"] / (rec["ms"] * 1e-3) / HBM_BPS
                rows.append(rec)
                print(json.dumps(rec))
    return rows


def onboarding():
    from sam6d_b200 import meshio
    from sam6d_b200.pipeline import SAM6D
    model = SAM6D(segmentor="fastsam", random_weights=True)
    u, v = np.meshgrid(np.linspace(0, 2 * np.pi, 41)[:-1], np.linspace(0.05, np.pi - 0.05, 21))
    verts = np.stack([60 * np.sin(v) * np.cos(u), 40 * np.sin(v) * np.sin(u), 30 * np.cos(v)], -1).reshape(-1, 3).astype(np.float32)
    faces = []
    for i in range(20):
        for j in range(40):
            a, b, c, d = i * 40 + j, i * 40 + (j + 1) % 40, (i + 1) * 40 + j, (i + 1) * 40 + (j + 1) % 40
            faces += [(a, c, b), (b, c, d)]
    mesh = meshio.Mesh(vertices=verts, faces=np.asarray(faces, np.int64), colors=np.full((len(verts), 3), 180, np.uint8))
    rows = []
    model.onboard(mesh, 512, rng=np.random.RandomState(0))                     # warm-up
    for level, dist in ((0, "all"), (1, "all"), (2, "all"), (2, "upper")):
        model.level_templates, model.pose_distribution = level, dist
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        ob = model.onboard(mesh, 512, rng=np.random.RandomState(0))
        torch.cuda.synchronize()
        rec = dict(level_templates=level, pose_distribution=dist, ism_views=int(ob.ref_cls.shape[0]), seconds=time.perf_counter() - t0,
                   peak_alloc_gb=(torch.cuda.max_memory_allocated() - before) / 1e9,
                   ref_patch_gb=ob.ref_patch.numel() * ob.ref_patch.element_size() / 1e9)
        del ob
        rows.append(rec)
        print(json.dumps(rec))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--onboard", action="store_true")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ism_score_bench needs a CUDA device")
    res = dict(card=card())
    print(json.dumps(res["card"]))
    res["scoring"] = scoring(args)
    if args.onboard:
        res["onboarding"] = onboarding()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
