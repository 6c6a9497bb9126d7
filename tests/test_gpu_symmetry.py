"""GPU: object symmetries (csrc/symmetry.cu, sam6d_b200/symmetry.py) and PEM hypotheses distinct up to them
(sam6d_coarse_pick_distinct_sym), against oracle/symmetry_oracle.py.

- Agreement counts equal the float64 oracle's except for queries whose float64 nearest distance lies within the oracle's
  derived fp32 bound of geo_tol (agreement_bound); colour decisions the same within 1e-5 of color_tol.
- The diameter within 8 u (relative) of the float64 brute force.
- find_symmetries on the GPU gives every procedural mesh's expected group, as built and moved off the origin under a rotation.
- The symmetric pick with identity-only ranges is ops.coarse_pick_distinct bit for bit on the arrays of a real forward; on a
  constructed cube set it skips 90-degree copies, matching the oracle's fp32 restatement, where the plain pick keeps them.
- End to end: symmetries=None gives today's records; "auto" runs, and the graph replays the launch-by-launch result.
- make_models_info's file is read back by bop.load_objects and bop_eval.load_models_info."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import pem_oracle as po
from oracle import symmetry_oracle as so

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _symmetry_meshes as sm                                                  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _t(a, dt=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)


def _rz(deg, axis=2):
    from sam6d_b200.bop_eval import _axis_angle
    return _axis_angle(np.eye(3)[axis], math.radians(deg))


# ---- kernels against the oracle ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("colour", [False, True])
def test_agreement_counts_against_the_oracle(colour):
    from sam6d_b200 import ops, symmetry
    rng = np.random.default_rng(1)
    mesh = sm.build("cube_colours")
    parts = symmetry._faces(mesh)
    q, qc = symmetry._sample(mesh, parts, 4096, rng, colour)
    tg, tc = symmetry._sample(mesh, parts, 32768, rng, colour)
    q, tg = np.float32(q), np.float32(tg)
    qc, tc = (np.float32(qc), np.float32(tc)) if colour else (None, None)
    rots = [np.eye(3), _rz(90), _rz(45), _rz(90, 0) @ _rz(180, 1), _rz(0.7, 1)]
    Rt = np.concatenate([np.stack([r.reshape(9) for r in rots]), rng.normal(0, 1.0, (len(rots), 3))], axis=1).astype(np.float32)
    Rt[0, 9:] = 0.0
    geo_tol, ctol = 2.5, 0.1
    count, sumsq = ops.symmetry_agreement(_t(Rt), _t(q), _t(tg), geo_tol, ctol, None if qc is None else _t(qc), None if tc is None else _t(tc))
    count, sumsq = count.cpu().numpy(), sumsq.cpu().numpy()
    want, ss64, ok, d, idx = so.agreement(Rt.astype(np.float64), q, qc, tg, tc, float(np.float32(geo_tol)), float(np.float32(ctol)))
    bound = so.agreement_bound(q, tg, Rt, geo_tol)
    for c in range(len(rots)):
        undecided = np.abs(d[c] - geo_tol) <= bound[c]
        if colour:
            cd = np.abs(qc - tc[idx[c]]).max(axis=1)
            undecided |= np.abs(cd - ctol) <= 1e-5
        lo = int((ok[c] & ~undecided).sum())
        hi = lo + int(undecided.sum())
        print(f"candidate {c}: gpu {count[c]} oracle {want[c]} undecided {int(undecided.sum())}")
        assert lo <= count[c] <= hi
        assert abs(sumsq[c] - ss64[c]) <= 1e-4 * ss64[c] + 1e-3


@pytest.mark.parametrize("V", [1, 2, 1000, 5000])
def test_diameter_against_brute_force(V):
    from sam6d_b200 import ops
    pts = np.random.default_rng(V).normal(0, 60.0, (V, 3)).astype(np.float32) + np.float32(200.0)
    d = math.sqrt(float(ops.point_diameter(_t(pts)).item()))
    want = so.diameter(pts)
    assert abs(d - want) <= 8 * U * want + 1e-12, (d, want)


def test_kernel_invalid_arguments():
    from sam6d_b200 import _lib, ops
    q = torch.zeros(4, 3, device="cuda")
    Rt = torch.zeros(1, 12, device="cuda")
    with pytest.raises(_lib.Sam6dError):
        ops.symmetry_agreement(Rt, q, q[:0], 1.0)                             # M = 0
    with pytest.raises(_lib.Sam6dError):
        ops.symmetry_agreement(Rt, q, q, float("nan"))
    with pytest.raises(_lib.Sam6dError):
        ops.point_diameter(q[:0])
    with pytest.raises(RuntimeError):
        ops.symmetry_agreement(Rt, q, q, 1.0, qc=q)                         # one colour set only


# ---- the finder ----------------------------------------------------------------------------------------------------------------
def _check_group(info, name, rot):
    nd, axis = sm.EXPECTED[name]
    assert len(info.get("symmetries_discrete", [])) == nd, (name, info)
    cont = info.get("symmetries_continuous", [])
    if axis is None:
        assert not cont
    else:
        assert len(cont) == 1
        want = rot @ np.asarray(axis)
        assert abs(abs(float(np.dot(cont[0]["axis"], want))) - 1.0) < 1e-3


@pytest.mark.parametrize("name", sm.NAMES)
def test_find_symmetries_on_the_gpu(name):
    from sam6d_b200 import bop_eval, symmetry
    for rot in (None, sm.random_rotation()):
        mesh = sm.build(name) if rot is None else sm.placed(sm.build(name), rot)
        info = symmetry.find_symmetries(mesh)
        _check_group(info, name, np.eye(3) if rot is None else rot)
        R, t = bop_eval.symmetry_transforms(info)
        nd, axis = sm.EXPECTED[name]
        assert len(R) == (1 + nd) * (1 if axis is None else 314)
        print(f"{name} {'rotated' if rot is not None else 'as built'}: {nd} discrete, continuous {axis is not None}")


# ---- the symmetric pick --------------------------------------------------------------------------------------------------------
def _coarse_arrays(monkeypatch, B=8):
    """the Rt, top and scores coarse_select sees in one real forward, and its radius"""
    from sam6d_b200 import ops
    from sam6d_b200.pem import Net
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
    monkeypatch.setattr(ops, "coarse_select", spy)
    g = torch.Generator(device="cuda").manual_seed(5)
    net(dict(dev), rand=torch.rand(B, po.N_PROPOSAL1 * 3, device="cuda", generator=g))
    rec["radius"] = ops.cloud_radius(dev["dense_po"])
    return rec


def test_identity_ranges_are_the_plain_pick(monkeypatch):
    from sam6d_b200 import ops
    a = _coarse_arrays(monkeypatch)
    B = a["Rt"].shape[0]
    symR = torch.eye(3, device="cuda").repeat(3, 1, 1)
    symt = torch.zeros(3, 3, device="cuda")
    ranges = torch.tensor([[b % 3, 1] for b in range(B)], dtype=torch.int32, device="cuda")
    for K, ang, dist in ((4, 30.0, 0.2), (16, 10.0, 0.05), (8, 90.0, 1.0)):
        plain = ops.coarse_pick_distinct(a["Rt"], a["top"], a["scores"], K, ang, dist)
        sym = ops.coarse_pick_distinct_sym(a["Rt"], a["top"], a["scores"], K, ang, dist, symR, symt, ranges, a["radius"])
        for x, y in zip(plain, sym):
            assert torch.equal(x, y), K
        print(f"K={K}: counts {plain[4].tolist()}")


def test_cube_pick_skips_symmetric_copies():
    from sam6d_b200 import ops, symmetry
    info = symmetry.find_symmetries(sm.build("cube"))
    R, t = symmetry.pick_set(info)
    assert len(R) == 24
    # hypothesis 1 is a pose; 2 and 3 are its 90-degree copies about the cube's axes; 4 is 45 degrees away (distinct)
    R1 = _rz(20, 0) @ _rz(-35, 1)
    t1 = np.array([0.1, -0.2, 3.0])
    poses = [(R1, t1), (R1 @ _rz(90), t1), (R1 @ _rz(90, 0), t1), (R1 @ _rz(45), t1), (R1 @ _rz(180, 1), t1 + 0.5)]
    n2 = len(poses)
    Rt = np.stack([np.concatenate([r.reshape(9), tt]) for r, tt in poses]).astype(np.float32)[None]
    scores = np.array([[0.9, 0.8, 0.7, 0.6, 0.5]], np.float32)
    top = np.arange(n2, dtype=np.int32)[None]
    radius = np.array([0.05], np.float32)
    rng = np.array([[0, len(R)]], np.int32)
    K = 4
    out = ops.coarse_pick_distinct_sym(_t(Rt), _t(top, torch.int32), _t(scores), K, 30.0, 0.2, _t(R.reshape(-1, 9)), _t(t),
                                       _t(rng, torch.int32), _t(radius))
    from sam6d_b200.ops import hypothesis_thresholds
    ct, dm = hypothesis_thresholds(30.0, 0.2)
    oR, ot, ov, oc = so.pick_distinct_sym(Rt, top, scores, K, ct, dm, R.reshape(-1, 9).astype(np.float32), t.astype(np.float32), rng, radius)
    assert np.array_equal(out[0].cpu().numpy(), oR) and np.array_equal(out[3].cpu().numpy(), ov) and np.array_equal(out[4].cpu().numpy(), oc)
    assert int(out[4][0]) == 3                                                  # 1, then 4 (45 degrees), then 5 (other place)
    plain = ops.coarse_pick_distinct(_t(Rt), _t(top, torch.int32), _t(scores), K, 30.0, 0.2)
    assert int(plain[4][0]) == 4                                                # the plain pick keeps the copies
    assert torch.equal(plain[0][0, 1], _t(Rt[0, 1, :9].reshape(3, 3)))
    assert torch.equal(out[0][0, 1], _t(Rt[0, 3, :9].reshape(3, 3)))


def test_pick_invalid_arguments(monkeypatch):
    from sam6d_b200 import _lib, ops
    Rt = torch.zeros(1, 4, 12, device="cuda")
    top = torch.zeros(1, 4, dtype=torch.int32, device="cuda")
    sc = torch.zeros(1, 4, device="cuda")
    symR, symt = torch.eye(3, device="cuda")[None], torch.zeros(1, 3, device="cuda")
    rng = torch.tensor([[0, 1]], dtype=torch.int32, device="cuda")
    rad = torch.ones(1, device="cuda")
    for kw in (dict(max_count=2049), dict(max_count=0)):
        with pytest.raises(_lib.Sam6dError):
            ops.coarse_pick_distinct_sym(Rt, top, sc, 2, 30.0, 0.2, symR, symt, rng, rad, **kw)
    with pytest.raises(_lib.Sam6dError):
        ops.coarse_pick_distinct_sym(Rt, top, sc, 5, 30.0, 0.2, symR, symt, rng, rad)      # K > n2


# ---- end to end ----------------------------------------------------------------------------------------------------------------
def test_end_to_end_with_symmetries(golden_dir):
    from test_gpu_icp import _sam6d, _scene_meshes
    model = _sam6d()
    meshes, frame = _scene_meshes(golden_dir)
    strip = lambda recs: [{k: v for k, v in r.items() if k != "time"} for r in recs]            # noqa: E731
    try:
        model.pem.set_hypotheses(4)
        base = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
        none = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0), symmetries=None)
        assert base.pose_inputs.symmetries is None and none.pose_inputs.symmetries is None
        res0 = model.detect_objects(*frame, base, rng=np.random.RandomState(5))
        res1 = model.detect_objects(*frame, none, rng=np.random.RandomState(5))
        assert res0.pem and strip(res0.pem) == strip(res1.pem)
        auto = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0), symmetries="auto")
        syms = auto.pose_inputs.symmetries
        assert syms is not None and tuple(syms.range.shape) == (2, 2)
        res = model.detect_objects(*frame, auto, rng=np.random.RandomState(5))
        assert len(res.pem) == len(res0.pem) and all(0 <= r["hypothesis"] < 4 for r in res.pem)
        print(f"auto symmetries: ranges {syms.range.tolist()}, hypotheses {[r['hypothesis'] for r in res.pem]}")
    finally:
        model.pem.set_hypotheses(1)


def test_graph_replay_with_symmetries():
    from sam6d_b200 import pipeline, symmetry
    from sam6d_b200.pem import Net
    net = Net().cuda().eval()
    net.load_state_dict(po.make_state_dict(seed=1), strict=True)
    net.set_precision("bf16").set_hypotheses(4)
    B = 4
    inp = po.make_inputs(B=B, n=2048, seed=3)
    data = {k: inp[k].cuda() for k in ("pts", "dense_fm", "dense_po", "dense_fo", "model")}
    infos = [symmetry.find_symmetries(sm.build("cube")), symmetry.find_symmetries(sm.build("cylinder"))]
    pipeline.symmetry_inputs(data, symmetry.pack_sets(infos, "cuda"), torch.tensor([0, 1, 0, 1], device="cuda"))
    g = torch.Generator(device="cuda").manual_seed(5)
    rand = torch.rand(B, po.N_PROPOSAL1 * 3, device="cuda", generator=g)
    keys = ("init_R", "init_t", "pred_R", "pred_t", "pred_pose_score", "hyp_init_R", "hyp_init_t", "hyp_valid", "hyp_index", "hyp_R")
    want = {k: v.clone() for k, v in net(dict(data), rand=rand).items() if k in keys}
    net.enable_graphs()
    for i in range(3):                                   # sighting, capture + replay, replay
        got = net(dict(data), rand=rand)
        for k in keys:
            assert torch.equal(got[k], want[k]), (i, k)
    assert net._graphs.replays == 2


# ---- make_models_info --------------------------------------------------------------------------------------------------------
def _write_ply(path, mesh):
    v, f = np.asarray(mesh.vertices), np.asarray(mesh.faces)
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(v), len(f)))
        for p in v:
            fh.write("%f %f %f\n" % tuple(p))
        for t in f:
            fh.write("3 %d %d %d\n" % tuple(t))


def test_make_models_info(tmp_path):
    from sam6d_b200 import bop, bop_eval
    from sam6d_b200.cli import make_models_info
    models = tmp_path / "ds" / "models"
    models.mkdir(parents=True)
    _write_ply(models / "obj_000001.ply", sm.build("cube"))
    _write_ply(models / "obj_000002.ply", sm.build("cylinder"))
    out = models / "models_info.json"
    assert make_models_info.main(["--cad_path", str(models / "obj_000001.ply"), str(models / "obj_000002.ply"), "--obj_ids", "1", "2",
                                  "--output", str(out)]) == 0
    info = bop_eval.load_models_info(str(out))
    assert len(info[1]["symmetries_discrete"]) == 23 and "symmetries_continuous" not in info[1]
    assert len(info[2]["symmetries_discrete"]) == 1 and len(info[2]["symmetries_continuous"]) == 1
    assert abs(info[1]["diameter"] - 80.0 * math.sqrt(3.0)) < 1e-3
    objs = bop.load_objects(str(tmp_path), "ds")
    assert objs.ids == [1, 2] and np.allclose(objs.diameters, [info[1]["diameter"] / 1000.0, info[2]["diameter"] / 1000.0])
    assert make_models_info.main(["--models_dir", str(models), "--output", str(tmp_path / "mi2.json")]) == 0
    assert json.load(open(tmp_path / "mi2.json")).keys() == json.load(open(out)).keys()
