"""tools/bop_run_bench.py -- times SAM6D.run_bop_ism and run_bop_pem on a synthetic BOP split built from the example frame
(640 x 480, two objects, seeded weights): per frame, the ISM's decoding and each stage of detect_objects, and the PEM's
decoding, instance building and Net.forward.  The device is synchronised at every stage mark, so the stage times add up.

    python tools/bop_run_bench.py [--frames 8] [--segmentor fastsam|sam] [--out bop_run_bench.json]

Prints one JSON object: the card, its power limit and max SM clock, and milliseconds per frame for each stage (the first
frame of each stage is a warm-up and is not counted)."""
import argparse
import importlib.util
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _split_builder():
    spec = importlib.util.spec_from_file_location("bop_split", os.path.join(ROOT, "tests", "test_gpu_bop.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._ycbv_split


class Stages:
    """mark(stage): synchronise, add the seconds since the previous mark to `stage` (after the warm-up frame)"""

    def __init__(self, frame_stage):
        self.t, self.acc, self.frames, self.frame_stage = time.perf_counter(), {}, 0, frame_stage

    def __call__(self, stage):
        torch.cuda.synchronize()
        now = time.perf_counter()
        if stage == self.frame_stage:
            self.frames += 1
        if self.frames >= 2:
            self.acc[stage] = self.acc.get(stage, 0.0) + (now - self.t)
        self.t = now

    def per_frame_ms(self):
        n = max(self.frames - 1, 1)
        return {k: round(v / n * 1e3, 3) for k, v in self.acc.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--segmentor", default="fastsam", choices=("fastsam", "sam"))
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bop_run_bench needs a CUDA device")
    from sam6d_b200.pipeline import SAM6D
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    tmp = tempfile.mkdtemp()
    try:
        root = _split_builder()(os.path.join(ROOT, "tests", "golden"), tmp)
        scene = os.path.join(root, "ycbv", "test", "000001")
        for k in range(1, args.frames):                                  # more frames of the same scene
            shutil.copy(os.path.join(scene, "rgb", "000000.png"), os.path.join(scene, "rgb", f"{k:06d}.png"))
            shutil.copy(os.path.join(scene, "depth", "000000.png"), os.path.join(scene, "depth", f"{k:06d}.png"))
        cams = json.load(open(os.path.join(scene, "scene_camera.json")))
        json.dump({str(k): cams["0"] for k in range(args.frames)}, open(os.path.join(scene, "scene_camera.json"), "w"))
        model = SAM6D(segmentor=args.segmentor, random_weights=True, confidence_thresh=-1)
        t0 = time.perf_counter()
        objects = model.onboard_bop(root, "ycbv", rng=np.random.RandomState(0))
        torch.cuda.synchronize()
        onboard_s = time.perf_counter() - t0
        ism = Stages("decode")
        det_path = os.path.join(tmp, "result_ycbv.json")
        recs = model.run_bop_ism(root, "ycbv", objects, det_path, max_frames=args.frames, mark=ism)
        for r in recs:                                                  # seeded weights score low: let every detection reach the PEM
            r["score"] = 0.5 + 0.5 * r["score"] if r["score"] > 0 else 0.5
        json.dump(recs, open(det_path, "w"))
        pem = Stages("decode")
        lines = model.run_bop_pem(det_path, root, "ycbv", os.path.join(root, "templates"), os.path.join(tmp, "result_ycbv.csv"),
                                  rng=np.random.RandomState(0), max_frames=args.frames + 1, mark=pem)
        res = {"gpu": smi, "segmentor": args.segmentor, "frames": args.frames, "image": "640x480", "objects": 2,
               "onboard_s": round(onboard_s, 2), "ism_detections_per_frame": len(recs) / max(args.frames, 1),
               "pem_poses_per_frame": len(lines) / max(args.frames, 1), "ism_ms_per_frame": ism.per_frame_ms(),
               "pem_ms_per_frame": pem.per_frame_ms()}
        res["ism_ms_per_frame"]["total"] = round(sum(res["ism_ms_per_frame"].values()), 3)
        res["pem_ms_per_frame"]["total"] = round(sum(res["pem_ms_per_frame"].values()), 3)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
