"""CPU: the multi-instance tracker's exclusive point assignment restated in numpy (tests/_track_scene_oracle.py) on small
hand-built frames and against the one-track selection of oracle/track_oracle.py; Tracker(max_instances > 1)'s start, merge
and slot rules with a stubbed SAM6D and stubbed device ops; the tracking CLI's new options."""
import inspect
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _track_scene_oracle as so  # noqa: E402
from oracle import track_oracle as to  # noqa: E402

F32 = np.float32
# fx = fy = 1, cx = cy = 0 and depth_scale 1000: z = raw exactly, and pixel (y, x) back-projects to (x z, y z, z) exactly
K1 = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])


def _frame(H, W, raw=1):
    return np.full((H, W), raw, np.uint16)


def _scene(rd, centre, radius, margin=0, raw=None):
    rd = np.asarray(rd, F32)
    raw = _frame(*rd.shape[1:]) if raw is None else raw
    return so.track_points_scene(rd, raw, 1000.0, K1, np.asarray(centre, F32), np.asarray(radius, F32), margin, 4)[3]


def test_front_rendered_track_wins():
    rd = np.zeros((2, 3, 3), F32)
    rd[0, 1, 1], rd[1, 1, 1] = 0.7, 0.5                                   # track 1 is in front at (1, 1)
    rd[0, 0, 0] = 0.3                                                     # only track 0 is rendered at (0, 0)
    cand = _scene(rd, np.zeros((2, 3)), [1e6, 1e6], margin=1)
    assert cand[1, 1, 1] and not cand[0, 1, 1]
    assert cand[0, 0, 0] and not cand[1, 0, 0]


def test_ineligible_front_track_does_not_take_the_pixel():
    rd = np.zeros((2, 3, 3), F32)
    rd[0, 1, 1], rd[1, 1, 1] = 0.2, 0.9
    # pixel (1, 1) is the point (1, 1, 1): outside track 0's gate about (10, 10, 10), inside track 1's
    centre = np.array([[10.0, 10.0, 10.0], [1.0, 1.0, 1.0]])
    cand = _scene(rd, centre, [1.0, 1.0])
    assert not cand[0, 1, 1] and cand[1, 1, 1]
    # a zero raw depth makes no track eligible
    raw = _frame(3, 3)
    raw[1, 1] = 0
    assert not _scene(rd, centre, [1.0, 1.0], raw=raw)[:, 1, 1].any()


def test_margin_band_goes_to_the_smaller_normalised_gate_distance():
    rd = np.zeros((2, 1, 5), F32)
    rd[0, 0, 0] = rd[1, 0, 4] = 1.0
    # pixel (0, 2) = (2, 0, 1) lies in both margin bands (m = 2), rendered by neither.  Track 0: d2 = 4, r = 4 (q = 0.25);
    # track 1: d2 = 1, r = 1.5 (q = 0.444): track 0 wins although track 1's centre is nearer
    centre = np.array([[2.0, 0.0, 3.0], [2.0, 0.0, 2.0]])
    cand = _scene(rd, centre, [4.0, 1.5], margin=2)
    assert cand[0, 0, 2] and not cand[1, 0, 2]
    # the front rule outranks the band: once track 1 is rendered there, it takes the pixel
    rd[1, 0, 2] = 5.0
    cand = _scene(rd, centre, [4.0, 1.5], margin=2)
    assert cand[1, 0, 2] and not cand[0, 0, 2]


def test_exact_ties_go_to_the_lower_track():
    rd = np.zeros((3, 1, 3), F32)
    rd[1, 0, 1] = rd[2, 0, 1] = 0.5                                        # equal rendered depth at (0, 1)
    rd[0, 0, 0] = 0.5
    cand = _scene(rd, np.zeros((3, 3)), [1e6, 1e6, 1e6], margin=1)
    assert cand[1, 0, 1] and not cand[2, 0, 1] and not cand[0, 0, 1]
    # equal normalised gate distance in the band: track 0 (its own silhouette at (0, 0)) and track 1 at pixel (0, 2)
    rd = np.zeros((2, 1, 3), F32)
    rd[0, 0, 0] = rd[1, 0, 0] = 1.0
    cand = _scene(rd, np.zeros((2, 3)), [10.0, 10.0], margin=2)
    assert cand[0, 0, 2] and not cand[1, 0, 2] and cand[0, 0, 0]


def _random_case(rng, L, H=24, W=29):
    rd = np.where(rng.rand(L, H, W) < 0.15, rng.uniform(0.5, 2.0, (L, H, W)), 0.0).astype(F32)
    rd[:, :, :3] = np.where(rng.rand(L, H, 3) < 0.3, F32(1.25), rd[:, :, :3])          # exact depth ties
    raw = rng.randint(0, 4, (H, W)).astype(np.uint16)
    K = np.array([[20.3, 0, 13.1], [0, 19.7, 11.2], [0, 0, 1]])
    centre = rng.uniform(-0.001, 0.004, (L, 3)).astype(F32)
    radius = rng.uniform(0.0005, 0.004, L).astype(F32)
    return rd, raw, K, centre, radius


@pytest.mark.parametrize("seed", range(6))
def test_every_pixel_is_a_candidate_of_at_most_one_track(seed):
    rng = np.random.RandomState(seed)
    rd, raw, K, centre, radius = _random_case(rng, 5)
    pts, count, index, cand = so.track_points_scene(rd, raw, 1.0, K, centre, radius, 2, 16)
    assert cand.sum(axis=0).max() <= 1 and cand.any()
    elig, _ = so.eligible(rd, raw, 1.0, K, centre, radius, 2)
    assert not (cand & ~elig).any()                                                     # only eligible tracks take pixels
    assert (cand.any(axis=0) == elig.any(axis=0)).all()                                 # and an eligible pixel is taken
    # where an eligible track is rendered, the pixel's track is an eligible rendered one with the least depth
    front = elig & (rd > 0)
    for y, x in zip(*np.nonzero(front.any(axis=0))):
        j = int(np.flatnonzero(cand[:, y, x])[0])
        assert front[j, y, x] and rd[j, y, x] == rd[front[:, y, x], y, x].min()
    assert count.tolist() == cand.reshape(5, -1).sum(axis=1).tolist()


@pytest.mark.parametrize("seed", range(6))
def test_one_track_equals_the_shared_rule(seed):
    rng = np.random.RandomState(100 + seed)
    rd, raw, K, centre, radius = _random_case(rng, 1)
    margin = int(rng.randint(0, 4))
    n = int(rng.choice([3, 16, 200]))
    a = so.track_points_scene(rd, raw, 1.0, K, centre, radius, margin, n)
    b = to.track_points(rd, raw, 1.0, K, centre, radius, margin, n)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y)


def test_merge_and_start_rules():
    # ids 4, 1, 7 with centroids: 1 at 0, 4 at 0.04 (within 0.05 of 1), 7 at 0.08 (0.08 from 1; its neighbour 4 is dropped)
    c = np.array([[0.04, 0, 0], [0.0, 0, 0], [0.08, 0, 0]])
    assert so.merge_drops([4, 1, 7], c, rho=0.1, assoc_scale=0.5) == {4}
    assert so.merge_drops([4, 1, 7], c, rho=0.1, assoc_scale=0.0) == set()
    s = np.array([0.2, 0.9, 0.5, 0.9, 0.35])
    cen = np.array([[0.5, 0, 0], [0.0, 0, 0], [0.2, 0, 0], [0.01, 0, 0], [0.3, 0, 0]])
    # no live track: the best (first of the equal 0.9s) starts; 3 is within 0.05 of it; 2 and 4 pass; 0 is below start_score
    assert so.starts(s, cen, [], 4, 0.1, 0.3, 0.5) == [1, 2, 4]
    assert so.starts(s, cen, [], 2, 0.1, 0.3, 0.5) == [1, 2]
    # with a live track at 0.21, 2 is too close; with none the best starts whatever its score
    assert so.starts(s, cen, [[0.21, 0, 0]], 4, 0.1, 0.3, 0.5) == [1, 4]
    assert so.starts([0.01], cen[:1], [], 1, 0.1, 0.3, 0.5) == [0]


# ---- Tracker(max_instances > 1), with stubs --------------------------------------------------------------------------------
class _StubSAM6D:
    """detect_objects returns `instances`, a list of (object, score, t metres) with R = I"""

    def __init__(self):
        self.device = torch.device("cpu")
        self.instances = []
        self.calls = 0

    def detect_objects(self, rgb, depth, cam_K, depth_scale, objects):
        self.calls += 1
        if not self.instances:
            return SimpleNamespace(frame=None, pem=[], R=None, t=None)
        obj = [o for o, _, _ in self.instances]
        scores = np.array([s for _, s, _ in self.instances])
        n = len(obj)
        R = torch.eye(3).repeat(n, 1, 1)
        t = torch.tensor([list(t) for _, _, t in self.instances], dtype=torch.float32)
        pem = [dict(scene_id=0, image_id=0, category_id=objects.obj_ids[o], bbox=[0, 0, 1, 1], score=float(s), time=0.0,
                    segmentation={"counts": [16], "size": [4, 4]}, R=R[i].tolist(), t=(t[i] * 1000).tolist())
               for i, (o, s) in enumerate(zip(obj, scores))]
        frame = SimpleNamespace(out={}, obj=np.array(obj), pose_scores=scores)
        return SimpleNamespace(frame=frame, pem=pem, R=R, t=t)


@pytest.fixture
def stubbed(monkeypatch):
    from sam6d_b200 import meshio, track
    script = {"inliers": {}, "shift": {}, "calls": []}

    def render_stub(meshes, poses, K, H, W):
        return {"depth": torch.zeros(len(meshes), 1, H, W)}

    def points_stub(name):
        def stub(rdepth, depth, depth_scale, K, centre, radius, margin, n):
            script["calls"].append(name)
            L, H, W = rdepth.shape
            return torch.zeros(L, n, 3), torch.full((L,), n, dtype=torch.int32), torch.ones(L, H, W, dtype=torch.uint8)
        return stub

    def icp_stub(R, t, pts, samples, normals, obj, radius, iters):
        # the ICP stub moves every track by +1 mm in x, and by script["shift"][z] where a track's z (mm) is listed
        o = obj.tolist()
        inl = torch.tensor([script["inliers"].get(round(float(t[j, 2]) * 1000), pts.shape[1]) for j in range(len(o))],
                           dtype=torch.int32)
        t1 = t.clone()
        t1[:, 0] += 0.001
        for j in range(len(o)):
            t1[j] += torch.tensor(script["shift"].get(round(float(t[j, 2]) * 1000), [0.0, 0.0, 0.0]))
        return R, t1, inl, torch.full((len(o),), 0.001), torch.full((len(o),), iters, dtype=torch.int32)

    def mask_rle_stub(masks):
        n, H, W = masks.shape
        return torch.zeros(n, dtype=torch.int32), torch.arange(n + 1, dtype=torch.int32)

    monkeypatch.setattr(track.render, "render", render_stub)
    monkeypatch.setattr(track.ops, "track_points", points_stub("track_points"))
    monkeypatch.setattr(track.ops, "track_points_scene", points_stub("track_points_scene"))
    monkeypatch.setattr(track.ops, "icp_refine", icp_stub)
    monkeypatch.setattr(track.ops, "mask_rle", mask_rle_stub)
    rng = np.random.RandomState(0)
    v = rng.normal(size=(20, 3)).astype(F32) * 30
    from scipy.spatial import ConvexHull
    meshes = [meshio.Mesh(vertices=v * s, faces=ConvexHull(v).simplices.astype(np.int64)) for s in (1.0, 0.5)]
    objects = SimpleNamespace(obj_ids=[3, 9], model_points_m=np.stack([m.vertices[:16] / 1000.0 for m in meshes]).astype(F32))
    return track, meshes, objects, script


RGB, DEPTH = np.zeros((4, 4, 3), np.uint8), np.ones((4, 4), np.uint16)


def _centroid(tr, o, t):
    return tr.centroid[o].numpy().astype(np.float64) + np.asarray(t, np.float64)        # R = I


def test_starts_follow_score_order_start_score_and_radius(stubbed):
    track, meshes, objects, script = stubbed
    sam = _StubSAM6D()
    tr = track.Tracker(sam, objects, meshes, max_instances=3, start_score=0.3, assoc_scale=0.5)
    rho = tr.rho
    d0 = 0.4 * rho[0]                                                      # within assoc_scale x rho of the first start
    sam.instances = [(0, 0.25, (0.3, 0.0, 1.0)), (0, 0.9, (0.0, 0.0, 1.0)), (0, 0.6, (d0, 0.0, 1.0)), (0, 0.5, (0.6, 0.0, 1.0)),
                     (0, 0.9, (-0.6, 0.0, 1.0)), (0, 0.7, (0.9, 0.0, 1.0)), (1, 0.1, (0.0, 0.5, 1.0))]
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)
    # the restated rule per object
    for o, slots in ((0, [0, 1, 2]), (1, [3, 4, 5])):
        rows = [i for i, ins in enumerate(sam.instances) if ins[0] == o]
        sc = np.array([sam.instances[i][1] for i in rows])
        cen = np.stack([_centroid(tr, o, sam.instances[i][2]) for i in rows])
        want = [rows[i] for i in so.starts(sc, cen, [], 3, rho[o], 0.3, 0.5)]
        got_t = [tuple(np.round(res.t[s].numpy().astype(np.float64), 6)) for s in slots if res.state[s] == "detected"]
        assert got_t == [tuple(np.round(np.asarray(sam.instances[i][2], np.float32).astype(np.float64), 6)) for i in want], o
    # object 0: the first 0.9 at x = 0, then the second 0.9 at x = -0.6, then 0.7 at 0.9; 0.6 is too close, full after three
    assert res.state == ["detected"] * 4 + ["absent"] * 2
    assert res.track_id.tolist() == [0, 1, 2, 3, -1, -1] and res.obj.tolist() == [0, 0, 0, 1, 1, 1]
    assert [r["score"] for r in res.records] == [0.9, 0.9, 0.7, 0.1]                      # object 1's one instance: score 0.1
    assert [r["track_id"] for r in res.records] == [0, 1, 2, 3]
    # a later detection fills object 1 only with instances that pass start_score and lie apart from its live track
    sam.instances = [(1, 0.29, (0.5, 0.5, 1.0)), (1, 0.3, (0.0012, 0.5, 1.0)), (1, 0.3, (0.5, 0.5, 1.0))]
    tr._since_detection = tr.redetect_interval
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)
    assert res.state == ["tracked"] * 4 + ["detected", "absent"]
    assert res.track_id.tolist() == [0, 1, 2, 3, 4, -1] and res.t[4].tolist() == pytest.approx([0.5, 0.5, 1.0])


def test_track_ids_are_never_reused(stubbed):
    track, meshes, objects, script = stubbed
    sam = _StubSAM6D()
    tr = track.Tracker(sam, objects, meshes, max_instances=2)
    assert tr.start(0, np.eye(3), [0.0, 0.0, 0.5]) == 0 and tr.start(0, np.eye(3), [0.3, 0.0, 0.6]) == 1
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)
    assert res.track_id.tolist() == [0, 1, -1, -1] and res.state == ["tracked", "tracked", "absent", "absent"]
    script["inliers"] = {500: 0}                                           # the track at z = 500 mm is lost
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)
    assert res.track_id.tolist() == [-1, 1, -1, -1] and res.state[0] == "absent" and tr.detection_due()
    script["inliers"] = {}
    sam.instances = [(0, 0.9, (0.0, 0.0, 0.5))]
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)                                  # detection restarts it in the lowest free slot
    assert res.track_id.tolist() == [2, 1, -1, -1] and res.state[:2] == ["detected", "tracked"]
    assert tr.start(1, np.eye(3), [0, 0, 1.0]) == 3
    tr.reset()
    assert tr.start(1, np.eye(3), [0, 0, 1.0]) == 0 and tr.track_id.tolist() == [-1, -1, 0, -1]


def test_merge_drops_the_younger_track_and_schedules_detection(stubbed):
    track, meshes, objects, script = stubbed
    sam = _StubSAM6D()
    tr = track.Tracker(sam, objects, meshes, max_instances=2, redetect_interval=100)
    rho = tr.rho[0]
    tr(RGB, DEPTH, K1.ravel(), 1.0)                                        # the first frame's detection (finds nothing)
    # slot 0 holds the younger track (id 1) once slot 1 is taken by id 0: free slot 0, keep id 0 in slot 1
    tr.start(0, np.eye(3), [0.0, 0.0, 0.7])
    tr.start(0, np.eye(3), [0.9, 0.0, 0.8])
    tr._drop(0)
    young = tr.start(0, np.eye(3), [0.9 + 0.8 * rho, 0.0, 0.801])          # slot 0, id 2, 0.8 rho from id 1 at first
    script["shift"] = {801: [-0.65 * rho, 0.0, 0.0]}
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)                                  # it moves to 0.15 rho of id 1: dropped
    assert young == 2 and res.state[:2] == ["absent", "tracked"] and res.track_id[:2].tolist() == [-1, 1]
    assert torch.isnan(res.R[0]).all() and res.inliers[0] == tr.n_points and res.detection is None
    assert [r["track_id"] for r in res.records] == [1]
    calls = sam.calls
    res = tr(RGB, DEPTH, K1.ravel(), 1.0)
    assert res.detection is not None and sam.calls == calls + 1
    # the restated rule on that frame's centroids
    c = np.stack([_centroid(tr, 0, [0.9 + 0.15 * rho + 0.001, 0, 0.801]), _centroid(tr, 0, [0.901, 0, 0.8])])
    assert so.merge_drops([2, 1], c, rho, 0.5) == {2}


def test_start_takes_the_lowest_free_slot_and_raises_when_full(stubbed):
    track, meshes, objects, script = stubbed
    tr = track.Tracker(_StubSAM6D(), objects, meshes, max_instances=3)
    assert [tr.start(1, np.eye(3), [0.1 * k, 0, 1]) for k in range(3)] == [0, 1, 2]
    assert tr.live.tolist() == [False] * 3 + [True] * 3
    with pytest.raises(ValueError):
        tr.start(1, np.eye(3), [0, 0, 1])
    tr._drop(4)
    assert tr.start(1, np.eye(3), [0, 0, 2]) == 3 and tr.track_id.tolist() == [-1, -1, -1, 0, 3, 2]
    # one instance per object: start replaces the object's track, as it always has
    one = track.Tracker(_StubSAM6D(), objects, meshes)
    assert one.start(0, np.eye(3), [0, 0, 1]) == 0 and one.start(0, np.eye(3), [0, 0, 2]) == 1
    assert one.track_id.tolist() == [1, -1] and one.t[0].tolist() == [0, 0, 2]


def test_one_instance_uses_the_shared_rule(stubbed):
    track, meshes, objects, script = stubbed
    sam = _StubSAM6D()
    sam.instances = [(0, 0.8, (0.0, 0.0, 0.5)), (0, 0.9, (0.5, 0.0, 0.5)), (1, 0.4, (0.0, 0.0, 0.7))]
    tr = track.Tracker(sam, objects, meshes)
    for _ in range(3):
        res = tr(RGB, DEPTH, K1.ravel(), 1.0)
    assert script["calls"] == ["track_points"] * 2
    assert res.state == ["tracked", "tracked"] and res.t[0].tolist() == pytest.approx([0.502, 0.0, 0.5])
    assert all("track_id" not in r for r in res.records)
    multi = track.Tracker(sam, objects, meshes, max_instances=2)
    script["calls"].clear()
    for _ in range(2):
        multi(RGB, DEPTH, K1.ravel(), 1.0)
    assert script["calls"] == ["track_points_scene"]


def test_cli_parses_the_instance_options(tmp_path):
    from sam6d_b200.cli import track_sam6d
    from sam6d_b200.track import Tracker
    base = ["--cad_path", "a.ply", "--rgb_dir", str(tmp_path), "--depth_dir", str(tmp_path), "--cam_path", "c.json", "--output_dir",
            str(tmp_path)]
    args = track_sam6d.get_parser().parse_args(base)
    sig = inspect.signature(Tracker).parameters
    for k in ("max_instances", "start_score", "assoc_scale"):
        assert getattr(args, k) == sig[k].default, k
    assert args.max_instances == 1
    args = track_sam6d.get_parser().parse_args(base + ["--max_instances", "3", "--start_score", "0.5", "--assoc_scale", "0.25"])
    assert (args.max_instances, args.start_score, args.assoc_scale) == (3, 0.5, 0.25)
