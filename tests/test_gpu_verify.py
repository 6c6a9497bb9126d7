"""GPU: the pose verification kernel (csrc/verify.cu through ops.verify_counts / ops.verify_poses) against the float64
restatement of oracle/verify_oracle.py, its ranking of right and wrong poses, and the pipeline's opt-in rescoring
(SAM6D(..., verify=True)).

Bounds.  u = 2^-24.  The kernel rounds dr = rdepth x rscale and e = do - dr to fp32, so its e is within u (|e| + 2 |dr|) of
the exact one (oracle.undecided); the oracle is fed the fp32 rscale and tau the kernel receives.  The silhouette and the mask
are exact, so n_sil and n_mask must match; every other count may differ from the oracle's by at most the hypothesis's number
of undecided pixels, whose total is printed."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import icp_oracle as io
from oracle import verify_oracle as vo

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_icp import _rot, bumpy_sphere_mm, hull_mesh_mm, _scene_meshes, _sam6d   # noqa: E402
from test_verify_cpu import TAU, hand_frame                                          # noqa: E402

pytestmark = pytest.mark.gpu

H, W, FX, CX, CY = 480, 640, 600.0, 320.0, 240.0
K = np.array([[FX, 0, CX], [0, FX, CY], [0, 0, 1.0]])
RSCALE = float(np.float32(1e-3))


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import ops as _ops
    return _ops


def _pose(R, t_m):
    p = np.eye(4, dtype=np.float32)
    p[:3, :3], p[:3, 3] = R, np.asarray(t_m, np.float32) * np.float32(1000.0)      # as verify_poses forms it, in fp32
    return p


def _render_depth(meshes, poses):
    """device meshes in mm, (n,4,4) poses with t in mm -> (n,H,W) f32 rendered depth in mm, rendered 32 at a time"""
    from sam6d_b200 import render
    out = []
    for i in range(0, len(poses), 32):
        p = torch.from_numpy(np.ascontiguousarray(poses[i:i + 32], dtype=np.float32))[:, None].cuda()
        out.append(render.render(meshes[i:i + 32], p, K, H, W)["depth"][:, 0])
    return torch.cat(out).contiguous()


def _scene(seed, occlusion=0.3):
    """the hull (object 0) at a known pose and a bumpy sphere (object 1, x 2) in front of it, hiding about `occlusion` of the
    hull's pixels -> (device meshes, true poses (R, t) of both, observed depth (H,W) f32 metres with 1 mm noise, masks (2,H,W)
    u8 = each object's visible pixels AND depth > 0, the hidden fraction)"""
    from sam6d_b200 import meshio, render
    rng = np.random.RandomState(seed)
    (v0, f0), (v1, f1) = hull_mesh_mm(os.path.join(os.path.dirname(__file__), "golden")), bumpy_sphere_mm(4)
    meshes = [render.upload(meshio.Mesh(vertices=v, faces=f.astype(np.int32))) for v, f in ((v0, f0), (v1 * 2.0, f1))]
    R0, t0 = _rot(rng), np.array([0.01, -0.02, 0.65])
    R1 = _rot(rng)
    d0 = _render_depth(meshes[:1], _pose(R0, t0)[None])[0]
    best = None
    for dx in np.linspace(0.0, 0.2, 21):                    # slide the occluder sideways until about `occlusion` is hidden
        t1 = t0 + np.array([dx, 0.0, -0.2])
        d1 = _render_depth(meshes[1:], _pose(R1, t1)[None])[0]
        hidden = float(((d0 > 0) & (d1 > 0) & (d1 < d0)).sum()) / float((d0 > 0).sum())
        if best is None or abs(hidden - occlusion) < abs(best[0] - occlusion):
            best = (hidden, t1, d1)
    hidden, t1, d1 = best
    z0, z1 = d0.double() / 1000.0, d1.double() / 1000.0
    front = torch.where((z0 > 0) & ((z1 == 0) | (z0 < z1)), z0, z1)
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    depth = torch.where(front > 0, front + 0.001 * torch.randn(front.shape, device="cuda", dtype=torch.float64, generator=g), front)
    depth = depth.float().contiguous()
    m0 = (z0 > 0) & ((z1 == 0) | (z0 < z1)) & (depth > 0)
    m1 = (z1 > 0) & ((z0 == 0) | (z1 <= z0)) & (depth > 0)
    masks = torch.stack([m0, m1]).to(torch.uint8).contiguous()
    return meshes, ((R0, t0), (R1, t1)), depth, masks, hidden


def _radius(meshes, o):
    return float(meshes[o].vertices.norm(dim=1).max()) / 1000.0


def _check_parity(ops, rdepth, depth, masks, mrow, tau, label):
    counts = ops.verify_counts(rdepth, depth, masks, mrow, tau, 1e-3).cpu().numpy()
    tau32 = np.asarray(tau, np.float32).astype(np.float64)
    dep, msk = depth.cpu().numpy(), masks.cpu().numpy()
    n_und = 0
    for p0 in range(0, len(mrow), 32):
        rd = rdepth[p0:p0 + 32].cpu().numpy()
        want = vo.counts(rd, dep, msk, mrow[p0:p0 + 32], tau32[p0:p0 + 32], RSCALE)
        und = vo.undecided(rd, dep, tau32[p0:p0 + 32], RSCALE).reshape(len(rd), -1).sum(axis=1)
        got = counts[p0:p0 + 32]
        assert np.array_equal(got[:, [0, 4]], want[:, [0, 4]]), label
        assert np.array_equal(got[:, 0], (rd > 0).reshape(len(rd), -1).sum(axis=1)), label        # the render's silhouette
        assert (np.abs(got[:, [1, 2, 3, 5]] - want[:, [1, 2, 3, 5]]) <= und[:, None]).all(), label
        n_und += int(und.sum())
    print(f"{label}: {n_und} undecided pixels of {len(mrow) * H * W}; counts {counts[:2].tolist()} ...")
    return counts


def test_hand_built_frame_is_exact(ops):
    rd, do, mask, _ = hand_frame()
    rd = np.concatenate([rd, rd * 0.5])                                            # a second hypothesis, also dyadic
    c = ops.verify_counts(torch.from_numpy(rd).cuda(), torch.from_numpy(do).cuda(), torch.from_numpy(mask).cuda(), [0, 0],
                          [TAU, TAU], 1.0).cpu().numpy()
    assert np.array_equal(c, vo.counts(rd, do, mask, [0, 0], [TAU, TAU], 1.0))
    assert c[0].tolist() == [9, 2, 4, 2, 7, 2]


@pytest.mark.parametrize("P", [1, 32, 200])
def test_parity_on_rendered_scenes(ops, P):
    meshes, ((R0, t0), (R1, t1)), depth, masks, hidden = _scene(P)
    rng = np.random.RandomState(100 + P)
    obj = (np.arange(P) % 5 == 4).astype(np.int64)                                  # one hypothesis in five is the occluder's
    poses = []
    for o in obj:
        R, t = (R0, t0) if o == 0 else (R1, t1)
        axis = rng.normal(size=3)
        Rp = R @ _rot(np.random.RandomState(rng.randint(1 << 30))) if rng.rand() < 0.1 else R
        Rp = Rp @ io.so3_exp(np.radians(rng.uniform(0, 20)) * axis / np.linalg.norm(axis))
        poses.append(_pose(Rp, t + rng.normal(scale=0.015, size=3)))
    rdepth = _render_depth([meshes[o] for o in obj], np.stack(poses))
    tau = np.asarray([rng.uniform(0.02, 0.15) * _radius(meshes, o) for o in obj], np.float32)
    mrow = np.where(rng.rand(P) < 0.8, obj, 1 - obj)
    _check_parity(ops, rdepth, depth, masks, mrow, tau, f"P={P} (hidden {hidden:.2f})")


def test_unaligned_and_odd_frames(ops):
    """the scalar path: an odd H x W, and a 480 x 640 frame whose rendered depths start 4 bytes off a 16-byte boundary,
    which must count what the vector path counts"""
    rng = np.random.RandomState(3)
    for h, w in ((37, 51), (1, 1)):
        rd = (rng.uniform(400, 800, size=(5, h, w)) * (rng.rand(5, h, w) < 0.7)).astype(np.float32)
        do = (rng.uniform(0.4, 0.8, size=(h, w)) * (rng.rand(h, w) < 0.9)).astype(np.float32)
        mk = (rng.rand(3, h, w) < 0.5).astype(np.uint8)
        tau = np.float32(rng.uniform(0.01, 0.2, 5))
        got = ops.verify_counts(torch.from_numpy(rd).cuda(), torch.from_numpy(do).cuda(), torch.from_numpy(mk).cuda(), [0, 2, 1, 1, 0],
                                tau, 1e-3).cpu().numpy()
        want = vo.counts(rd, do, mk, [0, 2, 1, 1, 0], tau.astype(np.float64), RSCALE)
        und = vo.undecided(rd, do, tau.astype(np.float64), RSCALE).reshape(5, -1).sum(axis=1)
        assert np.array_equal(got[:, [0, 4]], want[:, [0, 4]]) and (np.abs(got - want) <= und[:, None]).all()
    meshes, (true0, _), depth, masks, _ = _scene(7)
    rdepth = _render_depth([meshes[0]] * 3, np.stack([_pose(*true0)] * 3))
    buf = torch.empty(rdepth.numel() + 1, device="cuda")
    shifted = buf[1:].view(rdepth.shape)
    shifted.copy_(rdepth)
    assert shifted.data_ptr() % 16 != 0
    a = ops.verify_counts(rdepth, depth, masks, [0, 1, 0], [0.01] * 3)
    b = ops.verify_counts(shifted, depth, masks, [0, 1, 0], [0.01] * 3)
    assert torch.equal(a, b) and int(a[0, 2]) > 1000


def test_invalid_arguments_launch_nothing(ops):
    from sam6d_b200 import _lib
    P, M = 3, 2
    rd = torch.ones(P, 8, 8, device="cuda")
    do = torch.full((8, 8), 1e-3, device="cuda")                                  # = fp32(1 x fp32(1e-3)): e = 0, every pixel fits
    mk = torch.ones(M, 8, 8, dtype=torch.uint8, device="cuda")
    counts = torch.full((P, 6), -7, dtype=torch.int32, device="cuda")
    good_m, good_t = np.zeros(P, np.int32), np.full(P, 0.1, np.float32)

    def run(rd=rd, mrow=good_m, tau=good_t, P=P, M=M, h=8, w=8, rscale=1e-3, mask=mk):
        mrow, tau = np.ascontiguousarray(mrow, np.int32), np.ascontiguousarray(tau, np.float32)
        _lib.call("sam6d_pose_verify", rd, do, mask, mrow.ctypes.data, tau.ctypes.data, P, M, h, w, rscale, counts)

    bad = [dict(mrow=[0, 2, 0]), dict(mrow=[0, -1, 0]), dict(tau=[0.1, 0.0, 0.1]), dict(tau=[0.1, -1.0, 0.1]),
           dict(tau=[0.1, np.nan, 0.1]), dict(tau=[0.1, np.inf, 0.1]), dict(rscale=0.0), dict(rscale=float("nan")),
           dict(P=-1), dict(h=0), dict(w=0), dict(M=0), dict(rd=None), dict(mask=None)]
    for kw in bad:
        with pytest.raises(_lib.Sam6dError, match="invalid argument"):
            run(**kw)
    torch.cuda.synchronize()
    assert (counts == -7).all()
    run(P=0)                                                                       # nothing to do
    torch.cuda.synchronize()
    assert (counts == -7).all()
    run()
    assert counts.cpu().tolist() == [[64, 0, 64, 0, 64, 64]] * 3
    with pytest.raises(ValueError):
        ops.verify_counts(rd, do, mk, [0, 2, 0], 0.1)


def test_ranking(ops):
    """the true pose scores above wrong ones: 10 mm behind, 20 mm in front, rotated 15 degrees, flipped about the view axis and
    placed on the other object's segment; a hypothesis far behind everything is fully occluded and scores 0"""
    meshes, ((R0, t0), (R1, t1)), depth, masks, hidden = _scene(11)
    assert 0.2 < hidden < 0.4, hidden
    ray = t0 / np.linalg.norm(t0)
    axis = np.random.RandomState(12).normal(size=3)
    Rz = np.diag([-1.0, -1.0, 1.0])
    hyp = {"true": (R0, t0, 0), "10 mm behind": (R0, t0 + 0.010 * ray, 0), "20 mm in front": (R0, t0 - 0.020 * ray, 0),
           "15 deg rotated": (R0 @ io.so3_exp(np.radians(15) * axis / np.linalg.norm(axis)), t0, 0), "flipped": (Rz @ R0, t0, 0),
           "other segment": (R0, t1, 1), "fully occluded": (R0, t1 / np.linalg.norm(t1) * 6.0, 0)}
    names = list(hyp)
    R = torch.from_numpy(np.stack([hyp[k][0] for k in names]).astype(np.float32)).cuda()
    t = torch.from_numpy(np.stack([hyp[k][1] for k in names]).astype(np.float32)).cuda()
    mrow = [hyp[k][2] for k in names]
    tau = 0.1 * _radius(meshes, 0)
    counts, v = ops.verify_poses(R, t, [0] * len(names), meshes, depth, masks, mrow, K, tau)
    counts, v = counts.cpu().numpy(), v.cpu().numpy()
    for k, c, s in zip(names, counts, v):
        print(f"{k:>15}: verify {s:.4f}  counts {c.tolist()}")
    for i in range(1, len(names)):
        assert v[0] > v[i], names[i]
    occ = names.index("fully occluded")
    assert counts[occ, 0] > 0 and counts[occ, 2] == counts[occ, 3] == 0 and v[occ] == 0
    # the counts are those of the kernel on the renders: verify_poses is render.render + verify_counts
    rd = _render_depth([meshes[0]] * len(names), np.stack([_pose(hyp[k][0], hyp[k][1]) for k in names]))
    assert np.array_equal(ops.verify_counts(rd, depth, masks, mrow, tau).cpu().numpy(), counts)


def test_deterministic(ops):
    meshes, ((R0, t0), _), depth, masks, _ = _scene(13)
    rng = np.random.RandomState(14)
    R = torch.from_numpy(np.stack([R0 @ _rot(rng) if i % 2 else R0 for i in range(40)]).astype(np.float32)).cuda()
    t = torch.from_numpy((t0 + rng.normal(scale=0.01, size=(40, 3))).astype(np.float32)).cuda()
    a = ops.verify_poses(R, t, np.zeros(40, np.int64), meshes, depth, masks, np.zeros(40, np.int64), K, 0.01)
    b = ops.verify_poses(R, t, np.zeros(40, np.int64), meshes, depth, masks, np.zeros(40, np.int64), K, 0.01)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- the pipeline's opt-in rescoring ------------------------------------------------------------------------------------------
def _expected(ops, res, objs, frame_in):
    """ops.verify_poses of the reported poses against masks decoded again from the records' RLE"""
    from sam6d_b200 import inputs
    rgb, depth, cam_K, scale = frame_in
    fi = inputs.FrameInputs(res.pem, rgb, depth, cam_K, scale, 1.0)
    P = len(res.pem)
    tau = 0.1 * np.asarray(objs.radii, np.float64)[res.frame.obj]
    return ops.verify_poses(res.R.contiguous(), res.t.contiguous(), res.frame.obj, objs.pose_inputs.meshes, fi.depth, fi.mask, np.arange(P),
                            cam_K, tau)


def test_pipeline_frame_with_verification(ops, golden_dir):
    model = _sam6d()
    meshes, frame = _scene_meshes(golden_dir)
    try:
        objs_plain = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
        model.verify, model.icp_iters = True, 10
        objs = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
        assert objs_plain.pose_inputs.meshes is None and len(objs.pose_inputs.meshes) == 2
        assert torch.equal(objs.bank[1], objs_plain.bank[1]) and np.array_equal(objs.model_points_m, objs_plain.model_points_m)
        for icp_iters in (0, 10):
            model.icp_iters = icp_iters
            model.verify = False
            res0 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
            model.verify = True
            res1 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
            assert torch.equal(res0.R, res1.R) and torch.equal(res0.t, res1.t)
            drop = lambda recs, keys: [{k: v for k, v in r.items() if k not in keys} for r in recs]          # noqa: E731
            assert len(res1.pem) == len(res0.pem) > 0
            assert drop(res0.pem, ("time", "score")) == drop(res1.pem, ("time", "score", "verify"))
            assert all("verify" not in r for r in res0.pem) and "verify" not in res0.frame.out
            out0, out1 = res0.frame.out, res1.frame.out
            assert torch.equal(out0["pred_pose_score"], out1["pred_pose_score"])
            counts, v = _expected(ops, res1, objs, frame)
            assert torch.equal(counts, out1["verify_counts"]) and torch.equal(v, out1["verify"])
            want = (out1["pred_pose_score"] * out1["score"] * v).cpu().numpy()
            assert [r["score"] for r in res1.pem] == [float(x) for x in want]
            assert [r["verify"] for r in res1.pem] == [float(x) for x in v.cpu().numpy()]
            assert [r["score"] for r in res0.pem] == [float(x) for x in (out0["pred_pose_score"] * out0["score"]).cpu().numpy()]
            print(f"icp_iters {icp_iters}: {len(res1.pem)} poses, verify {[round(float(x), 4) for x in v.cpu().numpy()]}")
    finally:
        model.verify, model.icp_iters = False, 0


def test_run_sam6d_with_verify(golden_dir, tmp_path):
    import cv2
    import json
    from sam6d_b200.cli import run_sam6d
    meshes, (rgb, depth, K_, scale) = _scene_meshes(golden_dir)
    m = meshes[0]
    cad = str(tmp_path / "obj.ply")
    with open(cad, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\n"
                 "property uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                 % (len(m.vertices), len(m.faces)))
        for v, c in zip(m.vertices, m.colors):
            fh.write("%f %f %f %d %d %d\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
        for f in m.faces:
            fh.write("3 %d %d %d\n" % tuple(f))
    cv2.imwrite(str(tmp_path / "rgb.png"), rgb[:, :, ::-1])
    cv2.imwrite(str(tmp_path / "depth.png"), depth)
    json.dump(dict(cam_K=K_, depth_scale=scale), open(tmp_path / "camera.json", "w"))
    out = tmp_path / "out"
    assert run_sam6d.main(["--output_dir", str(out), "--cad_path", cad, "--rgb_path", str(tmp_path / "rgb.png"),
                           "--depth_path", str(tmp_path / "depth.png"), "--cam_path", str(tmp_path / "camera.json"),
                           "--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1", "--det_score_thresh", "-1",
                           "--template_size", "192", "--verify"]) == 0
    r = out / "sam6d_results"
    pem = json.load(open(r / "detection_pem.json"))
    print(f"run_sam6d --verify: {len(pem)} poses, verify {[round(x['verify'], 4) for x in pem]}")
    assert pem and all(0.0 <= x["verify"] <= 1.0 for x in pem) and (r / "vis_pem.png").exists()


def test_run_bop_pem_with_verification(golden_dir, tmp_path):
    import json
    import _bop_golden as bg
    gold = bg.load(golden_dir)
    split = str(tmp_path / "bop")
    os.makedirs(split)
    split = bg.write_split(gold, split)
    det_path = tmp_path / "dets.json"
    json.dump(gold["detections"], open(det_path, "w"))
    tdir = os.path.join(split, "BOP-Templates")
    model = _sam6d()
    try:
        l0 = model.run_bop_pem(str(det_path), split, "lmo", tdir, None, rng=np.random.RandomState(3))
        model.verify = True
        l1 = model.run_bop_pem(str(det_path), split, "lmo", tdir, None, rng=np.random.RandomState(3))
    finally:
        model.verify = False
    assert len(l0) == len(l1) == 12
    cols = lambda line: line.rstrip("\n").split(",")                      # noqa: E731
    # scene_id, im_id, obj_id, R and t equal; the score is multiplied by verify in [0, 1]; time is the host clock
    assert [cols(x)[:3] + cols(x)[4:6] for x in l0] == [cols(x)[:3] + cols(x)[4:6] for x in l1]
    s0, s1 = np.array([float(cols(x)[3]) for x in l0]), np.array([float(cols(x)[3]) for x in l1])
    assert (s1 <= s0 + 1e-6).all()
    print(f"run_bop_pem scores without / with verification: {s0.round(4).tolist()} / {s1.round(4).tolist()}")
