"""tools/make_golden_pn2.py -- writes tests/golden/pn2_ref.json: what the reference's own pointnet2._ext CUDA kernels return
for the seeded inputs of tests/test_gpu_pn2_ref.py, as the SHA-256 digest of each output plus 16 seeded elements.  Needs a GPU
and the reference extension built into oracle/_ref/ by oracle/build_ref_ext.py.

Usage: python tools/make_golden_pn2.py [out.json]"""
import importlib.util
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import build_ref_ext  # noqa: E402

# the cases and inputs are the test's own (loaded by path: tests/ is not a package)
_spec = importlib.util.spec_from_file_location("test_gpu_pn2_ref", os.path.join(ROOT, "tests", "test_gpu_pn2_ref.py"))
t = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(t)


def pack(out):
    out = out.cpu()
    idx = torch.randperm(out.numel(), generator=torch.Generator().manual_seed(0))[:16].sort()[0]
    return {"sha256": t.digest(out), "idx": idx.tolist(), "sample": out.reshape(-1)[idx].tolist()}


def main():
    ref = build_ref_ext.load_module()
    assert ref is not None, "oracle/_ref/ has no reference extension: run oracle/build_ref_ext.py where the reference sources are"
    gold = {}
    for b, n, m, dup in t.FPS_CASES:
        gold[f"fps/{b}/{n}/{m}/{int(dup)}"] = pack(ref.furthest_point_sampling(t.clouds(b, n, n + m, dup).cuda(), m))
    for b, n, m in t.FPS_BIG_CASES:
        gold[f"fps_big/{b}/{n}/{m}"] = pack(ref.furthest_point_sampling(t.clouds(b, n, n + m, dup=(n == 50000)).cuda(), m))
    for n, r, ns in t.BALL_CASES:
        x = t.clouds(3, n, n + ns).cuda()
        gold[f"ball/{n}/{r}/{ns}"] = pack(ref.ball_query(x, x, r, ns))
    pts, idx, gi = t.gather_inputs()
    gold["gather_points"] = pack(ref.gather_points(pts.cuda(), idx.cuda()))
    gold["group_points"] = pack(ref.group_points(pts.cuda(), gi.cuda()))
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "pn2_ref.json")
    with open(out, "w") as fh:
        fh.write("{\n" + ",\n".join(f" {json.dumps(k)}: {json.dumps(v, sort_keys=True)}" for k, v in sorted(gold.items())) + "\n}\n")
    print(f"wrote {out}: {torch.cuda.get_device_name()}, {len(gold)} entries")


if __name__ == "__main__":
    main()
