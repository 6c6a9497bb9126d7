"""CPU: the tracker's observed-point selection restated in numpy (oracle/track_oracle.py) on small hand-built frames; the
Tracker's detection schedule and loss rule with a stubbed SAM6D and stubbed device ops; the tracking CLI's frame pairing."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import track_oracle as to

F32 = np.float32
# fx = fy = 1, cx = cy = 0 and depth_scale 1000: z = raw exactly, and pixel (y, x) back-projects to (x z, y z, z) exactly
K1 = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])


def _frame(H, W, raw=1):
    return np.full((H, W), raw, np.uint16)


def test_dilation_is_a_square_window_clipped_at_the_border():
    H, W, m = 12, 10, 2
    rd = np.zeros((2, H, W), F32)
    rd[0, 5, 5] = 0.7
    rd[1, 0, 9] = 2.0                                                     # a corner pixel: the window is clipped
    cand = to.candidates(rd, _frame(H, W), 1000.0, K1, np.zeros((2, 3)), np.full(2, 1e6), m)
    want0 = np.zeros((H, W), bool)
    want0[3:8, 3:8] = True                                                # Chebyshev distance <= 2, distance 3 excluded
    want1 = np.zeros((H, W), bool)
    want1[0:3, 7:10] = True
    assert np.array_equal(cand[0], want0) and np.array_equal(cand[1], want1)
    # the two separable passes equal the direct 2-D window
    rng = np.random.RandomState(0)
    sil = rng.rand(3, 20, 17) < 0.05
    direct = np.zeros_like(sil)
    for o in range(3):
        for y, x in zip(*np.nonzero(sil[o])):
            direct[o, max(0, y - 3):y + 4, max(0, x - 3):x + 4] = True
    assert np.array_equal(to.dilate(sil, 3), direct)
    assert np.array_equal(to.dilate(sil, 0), sil)


def test_gate_boundary_is_inclusive():
    H, W = 4, 4
    rd = np.ones((3, H, W), F32)
    # pixel (2, 2) at z = 1 is (2, 2, 1): squared distance 9 from the origin; (3, 2) is 14
    r = np.array([3.0, np.nextafter(F32(3.0), F32(0.0)), -3.0], F32)
    cand = to.candidates(rd, _frame(H, W), 1000.0, K1, np.zeros((3, 3)), r, 0)
    assert cand[0, 2, 2] and not cand[0, 3, 2] and not cand[0, 2, 3]
    assert not cand[1, 2, 2] and cand[1, 2, 1]
    assert not cand[2].any()                                              # a non-positive radius admits nothing
    # a zero raw depth is never a candidate, a NaN centre admits nothing
    raw = _frame(H, W)
    raw[0, 0] = 0
    cand = to.candidates(rd[:1], raw, 1000.0, K1, np.full((1, 3), np.nan), np.array([100.0]), 0)
    assert not cand.any()
    cand = to.candidates(rd[:1], raw, 1000.0, K1, np.zeros((1, 3)), np.array([100.0]), 0)
    assert not cand[0, 0, 0] and cand[0].sum() == H * W - 1


def test_back_projection_is_float32_in_the_kernel_order():
    raw = np.array([[1234, 0], [65535, 7]], np.uint16)
    K = np.array([[612.3, 0, 318.9], [0, 611.7, 242.1], [0, 0, 1]])
    p = to.back_project(raw, 0.1, K)
    z = (raw.astype(F32) * F32(0.1)) / F32(1000.0)
    k = K.astype(F32)
    assert p.dtype == F32 and np.array_equal(p[..., 2], z)
    assert np.array_equal(p[1, 0, 0], ((F32(0) - k[0, 2]) * z[1, 0]) / k[0, 0])
    assert np.array_equal(p[1, 1, 1], ((F32(1) - k[1, 2]) * z[1, 1]) / k[1, 1])


def test_selection_in_raster_order():
    H, W = 6, 7
    rd = np.zeros((1, H, W), F32)
    rd[0, 1, 2] = rd[0, 4, 5] = 1.0
    raw = np.arange(1, H * W + 1, dtype=np.uint16).reshape(H, W)
    pts, count, index, cand = to.track_points(rd, raw, 1000.0, K1, np.zeros((1, 3)), np.array([1e9]), 1, 8)
    flat = np.flatnonzero(cand[0])
    assert count[0] == len(flat) == 18 and np.all(np.diff(flat) > 0)
    assert np.array_equal(index[0], flat[(np.arange(8) * 18) // 8])
    ys, xs = np.divmod(index[0], W)
    z = raw[ys, xs].astype(F32)
    assert np.array_equal(pts[0], np.stack([xs.astype(F32) * z, ys.astype(F32) * z, z], axis=1))


def test_fewer_candidates_than_points_wrap_and_none_give_zeros():
    H, W = 5, 5
    rd = np.zeros((2, H, W), F32)
    rd[0, 2, 2] = 1.0
    raw = _frame(H, W)
    raw[:, 1:] = 0                                                        # column 0 only: five pixels of object 0's window
    pts, count, index, _ = to.track_points(rd, raw, 1000.0, K1, np.zeros((2, 3)), np.full(2, 10.0), 2, 7)
    assert count.tolist() == [5, 0]
    assert index[0].tolist() == [0, 5, 10, 15, 20, 0, 5]
    assert (index[1] == -1).all() and not pts[1].any()
    assert to.select(5, 5).tolist() == [0, 1, 2, 3, 4] and to.select(10, 4).tolist() == [0, 2, 5, 7]


# ---- the Tracker's schedule and loss rule, with stubs ---------------------------------------------------------------------
class _StubSAM6D:
    """detect_objects returns, for every object listed in `found`, one PEM instance with score 0.5 + o / 10 (and a worse one)"""

    def __init__(self):
        self.device = torch.device("cpu")
        self.found = [0, 1]
        self.calls = 0

    def detect_objects(self, rgb, depth, cam_K, depth_scale, objects):
        self.calls += 1
        obj = [o for o in self.found for _ in range(2)]
        if not obj:
            return SimpleNamespace(frame=None, pem=[], R=None, t=None)
        n = len(obj)
        scores = np.array([0.5 + o / 10 - 0.2 * (i % 2) for i, o in enumerate(obj)])
        R = torch.eye(3).repeat(n, 1, 1)
        t = torch.tensor([[0.0, 0.0, 0.5 + i] for i in range(n)])
        pem = [dict(scene_id=0, image_id=0, category_id=objects.obj_ids[o], bbox=[0, 0, 1, 1], score=float(s), time=0.0,
                    segmentation={"counts": [16], "size": [4, 4]}, R=R[i].tolist(), t=(t[i] * 1000).tolist())
               for i, (o, s) in enumerate(zip(obj, scores))]
        frame = SimpleNamespace(out={}, obj=np.array(obj), pose_scores=scores)
        return SimpleNamespace(frame=frame, pem=pem, R=R, t=t)


@pytest.fixture
def stubbed(monkeypatch):
    from sam6d_b200 import meshio, track
    script = {"inliers": {}, "rms": {}}

    def render_stub(meshes, poses, K, H, W):
        return {"depth": torch.zeros(len(meshes), 1, H, W)}

    def track_points_stub(rdepth, depth, depth_scale, K, centre, radius, margin, n):
        L, H, W = rdepth.shape
        return torch.zeros(L, n, 3), torch.full((L,), n, dtype=torch.int32), torch.ones(L, H, W, dtype=torch.uint8)

    def icp_stub(R, t, pts, samples, normals, obj, radius, iters):
        o = obj.tolist()
        inl = torch.tensor([script["inliers"].get(i, pts.shape[1]) for i in o], dtype=torch.int32)
        rms = torch.tensor([script["rms"].get(i, 0.001) for i in o])
        return R, t + 0.001, inl, rms, torch.full((len(o),), iters, dtype=torch.int32)

    def mask_rle_stub(masks):
        n, H, W = masks.shape
        return torch.zeros(n, dtype=torch.int32), torch.arange(n + 1, dtype=torch.int32)

    monkeypatch.setattr(track.render, "render", render_stub)
    monkeypatch.setattr(track.ops, "track_points", track_points_stub)
    monkeypatch.setattr(track.ops, "icp_refine", icp_stub)
    monkeypatch.setattr(track.ops, "mask_rle", mask_rle_stub)
    rng = np.random.RandomState(0)
    v = rng.normal(size=(20, 3)).astype(F32) * 30
    from scipy.spatial import ConvexHull
    meshes = [meshio.Mesh(vertices=v * s, faces=ConvexHull(v).simplices.astype(np.int64)) for s in (1.0, 0.5)]
    objects = SimpleNamespace(obj_ids=[3, 9], model_points_m=np.stack([m.vertices[:16] / 1000.0 for m in meshes]).astype(F32))
    return track, meshes, objects, script


def test_tracker_schedule_and_loss_rule(stubbed):
    track, meshes, objects, script = stubbed
    sam = _StubSAM6D()
    tr = track.Tracker(sam, objects, meshes, redetect_interval=4, min_inlier_fraction=0.5, max_rms_m=0.005)
    rgb, depth = np.zeros((4, 4, 3), np.uint8), np.ones((4, 4), np.uint16)
    n = tr.n_points
    # frame -> (objects the ICP stub reports as failing with few inliers, with a large rms); objects the detector finds
    plan = {2: ({1}, set(), [0, 1]), 3: (set(), set(), []), 6: (set(), {0}, []), 9: (set(), set(), [0, 1])}
    first, lost_last, since = True, False, 0
    live = [False, False]
    for f in range(14):
        few, far, found = plan.get(f, (set(), set(), None))
        if found is not None:
            sam.found = found
        script["inliers"] = {o: n // 2 - 1 for o in few}
        script["rms"] = {o: 0.0051 for o in far}
        calls = sam.calls
        res = tr(rgb, depth, K1.ravel(), 1.0)
        # the restated rule: tracking of the live objects, then the schedule
        want = ["absent", "absent"]
        lost_now = False
        for o in range(2):
            if live[o]:
                inl, rms = script["inliers"].get(o, n), script["rms"].get(o, 0.001)
                if to.lost(inl, rms, n, 0.5, 0.005):
                    live[o], lost_now = False, True
                else:
                    want[o] = "tracked"
        due = to.detection_due(first, lost_last, since, 4)
        assert (res.detection is not None) == due == (sam.calls == calls + 1), f
        if due:
            since = 0
            for o in sam.found:
                if not live[o]:
                    live[o], want[o] = True, "detected"
        else:
            since += 1
        first, lost_last = False, lost_now
        assert res.state == want, (f, res.state, want)
        assert [r["track"] for r in res.records] == [s for s in want if s != "absent"]
        assert torch.isnan(res.R[[o for o in range(2) if want[o] == "absent"]]).all()
        assert torch.isfinite(res.R[[o for o in range(2) if want[o] != "absent"]]).all()
        for r in res.records:
            o = objects.obj_ids.index(r["category_id"])
            assert r["score"] == pytest.approx(0.5 + o / 10)                 # the detection that started the track
            assert set(r) >= {"scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation", "R", "t", "frames_tracked"}
    # the schedule above exercised every rule: first frame, loss, interval
    assert sam.calls >= 4


def test_tracker_start_and_reset(stubbed):
    track, meshes, objects, script = stubbed
    sam = _StubSAM6D()
    sam.found = []
    tr = track.Tracker(sam, objects, meshes)
    tr.start(1, np.eye(3), [0.0, 0.0, 0.7])
    res = tr(np.zeros((4, 4, 3), np.uint8), np.ones((4, 4), np.uint16), K1.ravel(), 1.0)
    assert res.state == ["absent", "tracked"] and res.detection is not None       # the first frame detects
    assert res.records[0]["frames_tracked"] == 1 and res.records[0]["t"] == pytest.approx([1.0, 1.0, 701.0])
    res = tr(np.zeros((4, 4, 3), np.uint8), np.ones((4, 4), np.uint16), K1.ravel(), 1.0)
    assert res.detection is None and res.records[0]["frames_tracked"] == 2
    tr.reset()
    assert not tr.live.any() and tr.detection_due()
    with pytest.raises(ValueError):
        track.Tracker(sam, objects, meshes[:1])


def test_loss_rule_thresholds():
    assert not to.lost(1024, 0.005, 2048, 0.5, 0.005)
    assert to.lost(1023, 0.001, 2048, 0.5, 0.005)
    assert to.lost(2048, 0.0050001, 2048, 0.5, 0.005)
    assert to.detection_due(False, False, 30, 30) and not to.detection_due(False, False, 29, 30)


def test_cli_pairs_frames_by_name(tmp_path):
    from sam6d_b200.cli import track_sam6d
    rgb, dep = tmp_path / "rgb", tmp_path / "depth"
    rgb.mkdir()
    dep.mkdir()
    for n in ("000010.png", "000002.png", "000001.png", "only_rgb.png"):
        (rgb / n).write_bytes(b"")
    for n in ("000002.png", "000010.png", "000001.png", "only_depth.png"):
        (dep / n).write_bytes(b"")
    assert track_sam6d.frame_pairs(str(rgb), str(dep)) == ["000001.png", "000002.png", "000010.png"]
    args = track_sam6d.get_parser().parse_args(["--cad_path", "a.ply", "b.ply", "--rgb_dir", str(rgb), "--depth_dir", str(dep),
                                                "--cam_path", "c.json", "--output_dir", str(tmp_path), "--segmentor_model",
                                                "fastsam", "--margin_px", "8", "--icp_iters", "3"])
    assert args.cad_path == ["a.ply", "b.ply"] and args.margin_px == 8 and args.icp_iters == 3 and args.redetect_interval == 30
    with pytest.raises(SystemExit):
        track_sam6d.main(["--cad_path", "a.ply", "--rgb_dir", str(rgb), "--depth_dir", str(tmp_path), "--cam_path", "c.json",
                          "--output_dir", str(tmp_path)])
    assert not os.path.exists(tmp_path / "sam6d_results")
