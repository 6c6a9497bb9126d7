"""GPU: the tracker's point selection (csrc/track.cu through ops.track_points) against oracle/track_oracle.py, and Tracker
(sam6d_b200/track.py) on rendered sequences of the 1.6 k-face hull mesh of tests/test_gpu_icp.py.

Bounds.  u = 2^-24.  The kernel's candidate set, counts and selected pixels are exact: every fp32 operation that decides
membership is rounded to nearest in the oracle's order, so they must be identical.  The points are checked twice: equal to
the oracle's float32 points, and within the fp32 rounding of the back-projection of the float64 formula
x = (u - cx) z / fx with z = raw s / 1000.  z is two roundings of exact operands plus the rounding of s to fp32: within
3u |z| (4u with slack).  x is three roundings on top of z's error and of fx's rounding (u relative each), so it is within
8u |x| plus the rounding of cx to fp32 carried through, u |cx| z / fx (2u with slack); the same for y."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import track_oracle as to  # noqa: E402
from oracle import icp_oracle as io  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
H, W = 480, 640
K = np.array([[600.0, 0.0, 319.5], [0.0, 600.0, 239.5], [0.0, 0.0, 1.0]])
DEPTH_SCALE = 1.0                                   # raw depth in mm
# a tracked pose must stay within these of the rendered ground truth at every frame.  The renderer samples pixel centres
# (x + 0.5) while the PEM's back-projection, which the tracker shares, uses x: about 0.5 mm of lateral bias at 0.6 m and
# f = 600, plus 1 mm depth noise and 1 mm quantisation averaged over ~2000 points
MAX_ROT_DEG, MAX_T_MM = 1.0, 2.0


def hull_mesh_mm(golden_dir):
    import test_gpu_icp
    return test_gpu_icp.hull_mesh_mm(golden_dir)


def _so3(axis, deg):
    a = np.asarray(axis, np.float64)
    return io.so3_exp(np.radians(deg) * a / np.linalg.norm(a))


def trajectory(n, deg=2.0, step_mm=5.0):
    """n ground-truth poses (R, t metres): 2 degrees about a fixed tilted axis and 5 mm along a fixed direction per frame"""
    R0 = _so3([0.3, -1.0, 0.4], 40.0)
    t0 = np.array([-0.04, 0.01, 0.6])
    d = np.array([1.0, 0.3, 0.5]) / np.linalg.norm([1.0, 0.3, 0.5])
    return [(R0 @ _so3([0.2, 1.0, -0.3], deg * f), t0 + d * step_mm * 1e-3 * f) for f in range(n)]


def _pose_mm(R, t):
    P = np.eye(4, dtype=np.float32)
    P[:3, :3], P[:3, 3] = R, np.asarray(t) * 1000.0
    return P


def render_depth_mm(meshes, poses):
    """render every (mesh, pose) into one depth map (the nearest surface), mm, float64"""
    from sam6d_b200 import render
    P = torch.from_numpy(np.stack([_pose_mm(R, t) for R, t in poses])[:, None]).cuda()
    d = render.render(meshes, P, K, H, W)["depth"][:, 0].cpu().numpy().astype(np.float64)
    d[d <= 0] = np.inf
    d = d.min(axis=0)
    d[np.isinf(d)] = 0.0
    return d


def raw_depth(depth_mm, rng, noise_mm=1.0, zero_frac=0.0):
    """mm depth -> u16 raw with Gaussian noise, 0 where nothing is seen and at a random zero_frac of the pixels"""
    raw = np.where(depth_mm > 0, np.rint(depth_mm + rng.normal(scale=noise_mm, size=depth_mm.shape)), 0.0)
    if zero_frac:
        raw[rng.rand(*raw.shape) < zero_frac] = 0.0
    return np.clip(raw, 0, 65535).astype(np.uint16)


def _meshes(golden_dir):
    from sam6d_b200 import meshio, render
    v, f = hull_mesh_mm(golden_dir)
    occ = meshio.Mesh(vertices=(v * 0.6).astype(np.float32), faces=f.astype(np.int32))
    main = meshio.Mesh(vertices=v.astype(np.float32), faces=f.astype(np.int32))
    return main, occ, [render.upload(m) for m in (main, occ)]


def _model_points(mesh, n=1024):
    from sam6d_b200 import meshio
    return (meshio.sample_surface(mesh.vertices, mesh.faces, n, np.random.RandomState(2)) / 1000.0).astype(np.float32)


# ---- kernel parity --------------------------------------------------------------------------------------------------------------
def parity_case(golden_dir, O, seed):
    """the hull at a ground-truth pose, a smaller hull in front of it, 1 mm noise and 2 % zero pixels; O predicted poses near
    the truth (one of them off-screen when O > 1) with their rendered depth and gates"""
    from sam6d_b200 import render
    rng = np.random.RandomState(seed)
    main, occ, up = _meshes(golden_dir)
    R, t = trajectory(1)[0]
    occ_pose = (_so3([1, 0, 0], 30), t + np.array([0.03, 0.0, -0.15]))
    raw = raw_depth(render_depth_mm(up, [(R, t), occ_pose]), rng, zero_frac=0.02)
    pred = []
    for o in range(O):
        Rp = R @ _so3(rng.normal(size=3), rng.uniform(0, 8))
        tp = t + rng.normal(scale=0.01, size=3)
        if O > 1 and o == O - 1:
            tp = t + np.array([2.0, 0.0, 0.0])                             # off-screen: no silhouette, no candidate
        pred.append((Rp, tp))
    P = torch.from_numpy(np.stack([_pose_mm(*p) for p in pred])[:, None]).cuda()
    rdepth = render.render([up[0]] * O, P, K, H, W)["depth"][:, 0].contiguous()
    mp = _model_points(main).astype(np.float64)
    c = mp.mean(0)
    gate_r = 1.5 * np.linalg.norm(mp - c, axis=1).max()
    centre = np.stack([Rp @ c + tp for Rp, tp in pred]).astype(np.float32)
    radius = np.full(O, gate_r, np.float32)
    return rdepth, raw, centre, radius


@pytest.mark.parametrize("O", [1, 21])
def test_points_match_the_oracle(golden_dir, O):
    from sam6d_b200 import ops
    rdepth, raw, centre, radius = parity_case(golden_dir, O, 3 + O)
    n, margin = 2048, 16
    pts, count, cand, index = ops.track_points(rdepth, torch.from_numpy(raw).cuda(), DEPTH_SCALE, K, torch.from_numpy(centre).cuda(),
                                               torch.from_numpy(radius).cuda(), margin, n, return_index=True)
    torch.cuda.synchronize()
    pts, count, cand, index = (x.cpu().numpy() for x in (pts, count, cand, index))
    p_o, c_o, i_o, cand_o = to.track_points(rdepth.cpu().numpy(), raw, DEPTH_SCALE, K, centre, radius, margin, n)
    assert np.array_equal(count, c_o), (count, c_o)
    assert np.array_equal(cand.astype(bool), cand_o)
    assert np.array_equal(index, i_o)
    assert np.array_equal(pts, p_o)
    if O > 1:
        assert count[-1] == 0 and (index[-1] == -1).all() and not pts[-1].any()
    assert (count[:O - 1 if O > 1 else 1] > n).all()
    # the float64 back-projection of the selected pixels, and the fp32 bound
    for o in range(O):
        if count[o] == 0:
            continue
        ys, xs = np.divmod(index[o].astype(np.int64), W)
        z = raw[ys, xs].astype(np.float64) * DEPTH_SCALE / 1000.0
        x = (xs - K[0, 2]) * z / K[0, 0]
        y = (ys - K[1, 2]) * z / K[1, 1]
        ref = np.stack([x, y, z], axis=1)
        bound = np.stack([8 * U * np.abs(x) + 2 * U * abs(K[0, 2]) * z / K[0, 0], 8 * U * np.abs(y) + 2 * U * abs(K[1, 2]) * z / K[1, 1],
                          4 * U * z], axis=1)
        assert (np.abs(pts[o] - ref) <= bound).all(), o
    print(f"O={O}: counts {count.tolist()}")


def test_points_edges(golden_dir):
    """margin 0 and a margin wider than the frame; fewer candidates than points (wrap); a zero-radius gate"""
    from sam6d_b200 import ops
    rdepth, raw, centre, radius = parity_case(golden_dir, 3, 9)
    radius[1] = 0.0
    _, _, _, cand0 = to.track_points(rdepth.cpu().numpy(), raw, DEPTH_SCALE, K, centre, radius, 16, 2048)
    keep = np.flatnonzero(cand0[0])[::97][:15]                             # 15 of object 0's candidates
    small = np.zeros_like(raw)
    small.reshape(-1)[keep] = raw.reshape(-1)[keep]
    for depth, margin in ((raw, 0), (raw, 5000), (small, 300)):
        args = (rdepth, torch.from_numpy(depth).cuda(), DEPTH_SCALE, K, torch.from_numpy(centre).cuda(), torch.from_numpy(radius).cuda(),
                margin, 2048)
        pts, count, cand, index = (x.cpu().numpy() for x in ops.track_points(*args, return_index=True))
        p_o, c_o, i_o, cand_o = to.track_points(rdepth.cpu().numpy(), depth, DEPTH_SCALE, K, centre, radius, margin, 2048)
        assert np.array_equal(count, c_o) and np.array_equal(index, i_o) and np.array_equal(pts, p_o), margin
        assert np.array_equal(cand.astype(bool), cand_o)
        assert count[1] == 0
    assert 0 < count[0] < 2048                                              # the last case wraps


# ---- sequences ------------------------------------------------------------------------------------------------------------------
class _NoDetector:
    """a SAM6D stand-in whose detections find nothing; counts its calls"""

    def __init__(self):
        self.device = torch.device("cuda")
        self.calls = 0

    def detect_objects(self, *args, **kwargs):
        self.calls += 1
        from types import SimpleNamespace
        return SimpleNamespace(frame=None, pem=[], R=None, t=None)


def sequence(golden_dir, n=30, occlude=(), seed=0):
    """n frames of the hull on trajectory(n) as raw u16 depth; the smaller hull passes in front in the frames of `occlude`"""
    rng = np.random.RandomState(seed)
    main, occ, up = _meshes(golden_dir)
    traj = trajectory(n)
    frames = []
    for f, (R, t) in enumerate(traj):
        poses = [(R, t)]
        if f in occlude:
            # 0.35 m from the camera, outside the gate, its image centre 120 .. 60 px left of the object's
            zo, off = 0.35, -120.0 + 15.0 * (f - min(occlude))
            u = K[0, 0] * t[0] / t[2] + off
            poses.append((_so3([1, 0, 0], 30), np.array([u * zo / K[0, 0], t[1] * zo / t[2], zo])))
            d = render_depth_mm(up, poses)
        else:
            d = render_depth_mm(up[:1], poses)
        frames.append(raw_depth(d, rng))
    return main, traj, frames


def _objects_of(mesh):
    from types import SimpleNamespace
    return SimpleNamespace(obj_ids=[1], model_points_m=_model_points(mesh)[None])


def run_sequence(golden_dir, frames, traj, main, **kw):
    from sam6d_b200.track import Tracker
    det = _NoDetector()
    tr = Tracker(det, _objects_of(main), [main], **kw)
    tr.start(0, traj[0][0], traj[0][1])
    rgb = np.zeros((H, W, 3), np.uint8)
    out = []
    for raw in frames:
        res = tr(rgb, raw, K.ravel(), DEPTH_SCALE)
        out.append(res)
    return out, det


def _errors(res, traj):
    e = []
    for r, (R, t) in zip(res, traj):
        Rg, tg = r.R[0].cpu().numpy().astype(np.float64), r.t[0].cpu().numpy().astype(np.float64)
        e.append((io.rotation_error_deg(Rg, R), 1000 * np.linalg.norm(tg - t)))
    return np.array(e)


@pytest.mark.parametrize("occlude", [(), tuple(range(12, 17))], ids=["clear", "occluded_5_frames"])
def test_sequence_follows_the_object(golden_dir, occlude):
    main, traj, frames = sequence(golden_dir, 30, occlude)
    hidden = 0.0
    if occlude:                                                            # the share of the object's pixels the occluder hides
        _, _, clear = sequence(golden_dir, 30)
        hidden = max(((clear[f] > 0) & (frames[f] > 0) & (frames[f] < 450)).sum() / (clear[f] > 0).sum() for f in occlude)
        assert hidden > 0.15
    res, det = run_sequence(golden_dir, frames, traj, main)
    err = _errors(res, traj)
    print(f"{'occluded' if occlude else 'clear'}: up to {100 * hidden:.0f} % hidden; max rotation error {err[:, 0].max():.3f} deg, "
          f"max translation error {err[:, 1].max():.3f} mm; inliers {[int(r.inliers[0]) for r in res]}; rms (mm) "
          f"{[round(1000 * float(r.rms[0]), 2) for r in res]}")
    assert all(r.state == ["tracked"] for r in res)
    assert det.calls == 1 and res[0].detection is not None                 # the first frame only
    assert (err[:, 0] < MAX_ROT_DEG).all() and (err[:, 1] < MAX_T_MM).all(), err
    assert [r.records[0]["frames_tracked"] for r in res] == list(range(1, 31))


def test_sequence_is_deterministic(golden_dir):
    main, traj, frames = sequence(golden_dir, 10)
    a, _ = run_sequence(golden_dir, frames, traj, main)
    b, _ = run_sequence(golden_dir, frames, traj, main)
    for x, y in zip(a, b):
        assert torch.equal(x.R, y.R) and torch.equal(x.t, y.t) and np.array_equal(x.inliers, y.inliers)


# ---- with the SAM6D pipeline ----------------------------------------------------------------------------------------------------
_MODEL = {}


def _sam6d():
    from sam6d_b200.pipeline import SAM6D
    if "m" not in _MODEL:
        _MODEL["m"] = SAM6D(segmentor="fastsam", random_weights=True, confidence_thresh=-1, det_score_thresh=-1)
    return _MODEL["m"]


def _onboard(model, main):
    from sam6d_b200 import meshio
    cols = np.random.RandomState(0).randint(40, 255, (len(main.vertices), 3)).astype(np.uint8)
    mesh = meshio.Mesh(vertices=main.vertices, faces=main.faces.astype(np.int64), colors=cols)
    return mesh, model.onboard_objects([mesh], obj_ids=[4], template_size=192, rng=np.random.RandomState(0))


def test_lost_track_triggers_detection(golden_dir):
    from sam6d_b200.track import Tracker
    model = _sam6d()
    main, traj, frames = sequence(golden_dir, 6)
    frames = frames[:3] + [np.zeros_like(frames[3])] * 3                  # the object leaves the view at frame 3
    mesh, objs = _onboard(model, main)
    rgb = np.zeros((H, W, 3), np.uint8)
    try:
        model.confidence_thresh = 2.0                                     # no proposal passes: detection finds nothing
        tr = Tracker(model, objs, [mesh])
        tr.start(0, traj[0][0], traj[0][1])
        res = [tr(rgb, raw, K.ravel(), DEPTH_SCALE) for raw in frames]
    finally:
        model.confidence_thresh = -1.0
    assert [r.state[0] for r in res] == ["tracked"] * 3 + ["absent"] * 3
    assert [r.detection is not None for r in res] == [True, False, False, False, True, False]
    assert res[4].detection.pem == [] and res[3].records == [] and res[4].records == []
    assert torch.isnan(res[5].R).all() and np.isnan(res[5].rms).all()


def test_detect_objects_unchanged_by_a_tracker(golden_dir):
    from sam6d_b200.track import Tracker
    model = _sam6d()
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    frame = (g["rgb"].numpy().astype(np.uint8), g["depth"].numpy().astype(np.uint16), g["cam_K"], g["depth_scale"])
    main, _, _ = _meshes(golden_dir)
    mesh, objs = _onboard(model, main)
    res0 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    tr = Tracker(model, objs, [mesh])
    np.random.seed(0)
    first = tr(*frame)
    np.random.seed(0)
    again = model.detect_objects(*frame, objs)
    res1 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    drop = lambda recs: [{k: v for k, v in r.items() if k != "time"} for r in recs]          # noqa: E731
    assert drop(res0.ism) == drop(res1.ism) and drop(res0.pem) == drop(res1.pem) and len(res0.pem) > 0
    assert torch.equal(res0.R, res1.R) and torch.equal(res0.t, res1.t)
    # the tracker's detection is detect_objects' result, and it starts the track from the best-scoring instance
    assert first.detection is not None and drop(first.detection.pem) == drop(again.pem)
    best = int(np.argmax(first.detection.frame.pose_scores))
    assert first.state == ["detected"] and torch.equal(first.R[0], first.detection.R[best])
    rec = first.records[0]
    assert rec["track"] == "detected" and rec["frames_tracked"] == 0 and rec["score"] == first.detection.pem[best]["score"]


def test_cli_writes_track_json(golden_dir, tmp_path):
    import cv2
    from test_gpu_cli import _write_ply
    from sam6d_b200.cli import track_sam6d
    main, traj, frames = sequence(golden_dir, 3)
    rgb_dir, depth_dir = tmp_path / "rgb", tmp_path / "depth"
    rgb_dir.mkdir()
    depth_dir.mkdir()
    for i, raw in enumerate(frames):
        rgb = np.full((H, W, 3), 80, np.uint8)
        rgb[raw > 0] = (200, 120, 40)
        cv2.imwrite(str(rgb_dir / f"{i:06d}.png"), rgb)
        cv2.imwrite(str(depth_dir / f"{i:06d}.png"), raw)
    cad = str(tmp_path / "obj.ply")
    _write_ply(cad, main.vertices, main.faces, np.random.RandomState(0).randint(40, 255, (len(main.vertices), 3)))
    json.dump(dict(cam_K=K.ravel().tolist(), depth_scale=DEPTH_SCALE), open(tmp_path / "camera.json", "w"))
    out = tmp_path / "out"
    np.random.seed(0)
    assert track_sam6d.main(["--cad_path", cad, "--rgb_dir", str(rgb_dir), "--depth_dir", str(depth_dir), "--cam_path",
                             str(tmp_path / "camera.json"), "--output_dir", str(out), "--segmentor_model", "fastsam",
                             "--random_weights", "--template_size", "192", "--confidence_thresh", "-1", "--det_score_thresh",
                             "-1"]) == 0
    res = json.load(open(out / "sam6d_results" / "track_pem.json"))
    assert [r["frame"] for r in res] == ["000000.png", "000001.png", "000002.png"]
    keys = {"scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation", "R", "t", "track", "frames_tracked"}
    for r in res:
        assert isinstance(r["records"], list) and len(r["records"]) <= 1
        for rec in r["records"]:
            assert set(rec) == keys and rec["category_id"] == 1 and rec["track"] in ("tracked", "detected")
            R = np.array(rec["R"])
            assert R.shape == (3, 3) and np.allclose(R @ R.T, np.eye(3), atol=1e-4) and len(rec["t"]) == 3
            assert rec["segmentation"]["size"] == [H, W]
    print("CLI states:", [[rec["track"] for rec in r["records"]] for r in res])
