"""Time the symmetry finder and the symmetric hypothesis pick on the GPU (sam6d_b200/symmetry.py, csrc/symmetry.cu).

    python tools/symmetry_bench.py [--out result.json]

- find_symmetries on closed n-gon prisms of about 1e4, 1e5 and 5e5 vertices (their group: an n-fold axis, n > 12, so the axis
  is reported continuous): the device time of each stage's ops.symmetry_agreement call (CUDA events around it), the number of
  candidates and the point pairs it tests, and the whole call on the host clock (sampling and candidate axes included).
- ops.point_diameter on the prisms' vertices, CUDA events over 5 calls.
- ops.coarse_pick_distinct and ops.coarse_pick_distinct_sym (the cube's 24 transforms, the cylinder's 146) on the arrays of a
  real B = 32 forward at K = 4, CUDA events over 200 launches each.
Prints the card's name, power limit and maximum SM clock, then one JSON line."""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from hypotheses_bench import card, events  # noqa: E402


class TimedBackend:
    """symmetry.GpuBackend that records each agreement call's device time, candidates and point pairs"""

    def __init__(self):
        from sam6d_b200 import symmetry
        self.gpu = symmetry.GpuBackend()
        self.calls = []

    def agreement(self, Rt, q, qc, tg, tc, geo_tol, color_tol):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.gpu.agreement(Rt, q, qc, tg, tc, geo_tol, color_tol)
        e1.record()
        torch.cuda.synchronize()
        C = len(Rt)
        self.calls.append(dict(candidates=C, pairs=C * len(q) * len(tg), ms=e0.elapsed_time(e1)))
        return out

    def diameter(self, pts):
        return self.gpu.diameter(pts)


def finder(n_seg):
    from sam6d_b200 import ops, symmetry
    import _symmetry_meshes as sm
    mesh = sm.prism(n_seg, 40.0, 90.0)
    V = len(mesh.vertices)
    be = TimedBackend()
    symmetry.find_symmetries(mesh, backend=be)                 # warm-up: module load, allocator
    be.calls = []
    t0 = time.perf_counter()
    info = symmetry.find_symmetries(mesh, backend=be)
    total = 1000.0 * (time.perf_counter() - t0)
    pts = torch.from_numpy(np.asarray(mesh.vertices, np.float32)).cuda()
    dia = events(lambda: ops.point_diameter(pts), 5)
    return dict(vertices=V, stages=be.calls, find_ms=total, diameter_ms=dia, diameter_pairs=V * (V - 1) // 2,
                discrete=len(info.get("symmetries_discrete", [])), continuous=len(info.get("symmetries_continuous", [])))


def pick():
    from sam6d_b200 import ops, pipeline, symmetry
    from oracle import pem_oracle as po
    from sam6d_b200.pem import Net
    import _symmetry_meshes as sm
    B, K = 32, 4
    net = Net().cuda().eval()
    net.load_state_dict(po.make_state_dict(seed=1), strict=True)
    inp = po.make_inputs(B=B, n=2048, seed=3)
    dev = {k: inp[k].cuda() for k in ("pts", "dense_fm", "dense_po", "dense_fo", "model")}
    rec = {}
    real = ops.coarse_select

    def spy(Rt, top, *a):
        out = real(Rt, top, *a)
        rec.update(Rt=Rt.clone(), top=top.clone(), scores=out[2].clone())
        return out
    ops.coarse_select = spy
    try:
        net(dict(dev), rand=torch.rand(B, po.N_PROPOSAL1 * 3, device="cuda"))
    finally:
        ops.coarse_select = real
    radius = ops.cloud_radius(dev["dense_po"])
    res = dict(B=B, K=K, plain_us=1000.0 * events(lambda: ops.coarse_pick_distinct(rec["Rt"], rec["top"], rec["scores"], K, 30.0, 0.2), 200))
    for name in ("cube", "cylinder"):
        s = symmetry.pack_sets([symmetry.find_symmetries(sm.build(name))], "cuda")
        rng = s.range[torch.zeros(B, dtype=torch.int64, device="cuda")].contiguous()
        res[f"sym_{name}_S"] = int(s.R.shape[0])
        res[f"sym_{name}_us"] = 1000.0 * events(lambda: ops.coarse_pick_distinct_sym(rec["Rt"], rec["top"], rec["scores"], K, 30.0, 0.2,
                                                                                    s.R, s.t, rng, radius), 200)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(card())
    res = dict(card=card(), finder=[finder(n) for n in (4999, 49999, 249999)], pick=pick())
    for f in res["finder"]:
        st = ", ".join(f"{c['candidates']} cand {c['ms']:.1f} ms ({c['pairs'] / c['ms'] / 1e9:.1f} Gpair/ms)" for c in f["stages"])
        print(f"V = {f['vertices']}: find_symmetries {f['find_ms']:.0f} ms [{st}]; diameter {f['diameter_ms']:.2f} ms "
              f"({f['diameter_pairs'] / 1e9:.2f} G pairs); {f['discrete']} discrete, {f['continuous']} continuous")
    p = res["pick"]
    print(f"pick B={p['B']} K={p['K']}: plain {p['plain_us']:.1f} us, sym cube (S={p['sym_cube_S']}) {p['sym_cube_us']:.1f} us, "
          f"sym cylinder (S={p['sym_cylinder_S']}) {p['sym_cylinder_us']:.1f} us")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
