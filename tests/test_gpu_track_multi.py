"""GPU: the exclusive point assignment of several tracks (csrc/track.cu at sam6d_track_points_scene, ops.track_points_scene)
against tests/_track_scene_oracle.py, and Tracker(max_instances > 1) (sam6d_b200/track.py) on rendered sequences of two copies
of the 1.6 k-face hull mesh of tests/test_gpu_icp.py (radius about 115 mm).

The candidate sets, counts, selected pixels and points are exact (every fp32 operation that decides membership is rounded to
nearest in the oracle's order), so they must be identical to the oracle's; the points' fp32 bound against the float64
back-projection is tests/test_gpu_track.py's and is not repeated here.  A tracked pose must stay within the bound of
tests/test_gpu_track.py's sequences, 1 degree and 2 mm, of its own copy."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _track_scene_oracle as so  # noqa: E402
import test_gpu_track as tt  # noqa: E402
from oracle import icp_oracle as io  # noqa: E402

pytestmark = pytest.mark.gpu

H, W, K, DEPTH_SCALE = tt.H, tt.W, tt.K, tt.DEPTH_SCALE
N, MARGIN = 2048, 16


def _gate(main):
    mp = tt._model_points(main).astype(np.float64)
    c = mp.mean(0)
    return c, 1.5 * np.linalg.norm(mp - c, axis=1).max()


def _cuda(*a):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


def _run_both(rdepth, raw, centre, radius, margin=MARGIN, n=N):
    """the kernel's and the oracle's outputs, as numpy"""
    from sam6d_b200 import ops
    d, c, r = _cuda(raw, centre, radius)
    pts, count, cand, index = (x.cpu().numpy() for x in ops.track_points_scene(rdepth, d, DEPTH_SCALE, K, c, r, margin, n,
                                                                                  return_index=True))
    ref = so.track_points_scene(rdepth.cpu().numpy(), raw, DEPTH_SCALE, K, centre, radius, margin, n)
    return (pts, count, index, cand.astype(bool)), ref


def _assert_equal(got, ref, what=""):
    for name, g, r in zip(("pts", "count", "index", "cand"), got, ref):
        assert np.array_equal(g, r), (what, name)


# ---- kernel parity --------------------------------------------------------------------------------------------------------------
def scene_case(golden_dir, n_objects, copies, seed, spread=True):
    """n_objects x copies copies of the hull: the truth spread over the frame (or overlapping around the centre) at 0.55 -
    0.9 m, rendered with 1 mm noise and 2 % zero pixels; one predicted pose per copy near its truth, with its rendered depth
    and gate (L = n_objects x copies tracks)"""
    from sam6d_b200 import render
    rng = np.random.RandomState(seed)
    main, _, up = tt._meshes(golden_dir)
    truth = []
    for _ in range(n_objects * copies):
        z = 0.55 + 0.35 * rng.rand()
        u, v = (rng.uniform(120, 520), rng.uniform(100, 380)) if spread else (rng.uniform(260, 380), rng.uniform(200, 280))
        truth.append((tt._so3(rng.normal(size=3), rng.uniform(0, 180)), np.array([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z])))
    raw = tt.raw_depth(tt.render_depth_mm([up[0]] * len(truth), truth), rng, zero_frac=0.02)
    pred = [(R @ tt._so3(rng.normal(size=3), rng.uniform(0, 5)), t + rng.normal(scale=0.005, size=3)) for R, t in truth]
    P = torch.from_numpy(np.stack([tt._pose_mm(*p) for p in pred])[:, None]).cuda()
    rdepth = render.render([up[0]] * len(pred), P, K, H, W)["depth"][:, 0].contiguous()
    c, gate_r = _gate(main)
    centre = np.stack([R @ c + t for R, t in pred]).astype(np.float32)
    return rdepth, raw, centre, np.full(len(pred), gate_r, np.float32)


def _overlaps(rd, cand, elig):
    """(pixels taken by two or more tracks, pixels a track takes while another eligible track is rendered in front there)"""
    shared = int((cand.sum(axis=0) > 1).sum())
    z = np.where(rd > 0, rd, np.inf)
    front = np.where(elig & (rd > 0), z, np.inf).min(axis=0)                # the nearest eligible rendered surface
    behind = cand & (z > front[None])
    return shared, int(behind.any(axis=0).sum())


def test_two_overlapping_copies_match_the_oracle(golden_dir):
    rdepth, raw, centre, radius = scene_case(golden_dir, 1, 2, 11, spread=False)
    got, ref = _run_both(rdepth, raw, centre, radius)
    _assert_equal(got, ref)
    rd = rdepth.cpu().numpy()
    both = ((rd > 0).all(axis=0)).sum()
    assert both > 1000 and (got[1] > N).all() and got[3].sum(axis=0).max() == 1
    print(f"L=2: counts {got[1].tolist()}, {both} pixels rendered by both")


def test_42_tracks_match_the_oracle_and_never_share(golden_dir):
    from sam6d_b200 import ops
    rdepth, raw, centre, radius = scene_case(golden_dir, 21, 2, 42)
    got, ref = _run_both(rdepth, raw, centre, radius)
    _assert_equal(got, ref)
    rd = rdepth.cpu().numpy()
    elig, _ = so.eligible(rd, raw, DEPTH_SCALE, K, centre, radius, MARGIN)
    d, c, r = _cuda(raw, centre, radius)
    shared_cand = ops.track_points(rdepth, d, DEPTH_SCALE, K, c, r, MARGIN, N)[2].cpu().numpy().astype(bool)
    s_shared, s_behind = _overlaps(rd, shared_cand, elig)
    m_shared, m_behind = _overlaps(rd, got[3], elig)
    overlap = int(((rd > 0).sum(axis=0) > 1).sum())
    print(f"L=42: {overlap} pixels rendered by two or more tracks; track_points: {s_shared} pixels shared, {s_behind} taken behind "
          f"another track's rendered front; track_points_scene: {m_shared}, {m_behind}; counts {got[1].tolist()}")
    assert overlap > 0 and s_shared > 0
    assert m_shared == 0 and m_behind == 0
    # every pixel the shared rule gives to some track goes to exactly one track here
    assert np.array_equal(got[3].any(axis=0), shared_cand.any(axis=0))


def test_edges(golden_dir):
    """L = 1 equals track_points; margin 0; W not a multiple of 256; a track with an empty render; wrap; no candidates"""
    from sam6d_b200 import ops
    rdepth, raw, centre, radius = scene_case(golden_dir, 1, 3, 5, spread=False)
    for j in range(3):
        d, c, r = _cuda(raw, centre[j:j + 1], radius[j:j + 1])
        one = rdepth[j:j + 1].contiguous()
        a = ops.track_points_scene(one, d, DEPTH_SCALE, K, c, r, MARGIN, N, return_index=True)
        b = ops.track_points(one, d, DEPTH_SCALE, K, c, r, MARGIN, N, return_index=True)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), j
    base, ref = _run_both(rdepth, raw, centre, radius)
    _assert_equal(base, ref, "margin 16")
    got, ref = _run_both(rdepth, raw, centre, radius, margin=0)
    _assert_equal(got, ref, "margin 0")
    Wc = 600                                                               # columns 0 .. 599 only
    got, ref = _run_both(rdepth[:, :, :Wc].contiguous(), np.ascontiguousarray(raw[:, :Wc]), centre, radius)
    _assert_equal(got, ref, "W = 600")
    empty = rdepth.clone()
    empty[1] = 0.0                                                         # track 1 renders nothing
    got, ref = _run_both(empty, raw, centre, radius)
    _assert_equal(got, ref, "empty render")
    assert got[1][1] == 0 and (got[2][1] == -1).all() and not got[0][1].any()
    keep = np.flatnonzero(base[3][0])[::101][:20]                          # 20 of track 0's candidates: fewer than N
    small = np.zeros_like(raw)
    small.reshape(-1)[keep] = raw.reshape(-1)[keep]
    got, ref = _run_both(rdepth, small, centre, radius)
    _assert_equal(got, ref, "wrap")
    assert 0 < got[1][0] < N
    got, ref = _run_both(rdepth, np.zeros_like(raw), centre, radius)
    _assert_equal(got, ref, "no candidates")
    assert (got[1] == 0).all() and (got[2] == -1).all()


def test_invalid_arguments_return_minus_22(golden_dir):
    from sam6d_b200 import _lib
    L, h, w = 2, 8, 8
    rd = torch.ones(L, h, w, device="cuda")
    depth = torch.ones(h, w, dtype=torch.uint16, device="cuda")
    centre, radius = torch.zeros(L, 3, device="cuda"), torch.ones(L, device="cuda")
    hm, dm, cand = (torch.full((L, h, w), 7, dtype=torch.uint8, device="cuda") for _ in range(3))
    rows = torch.full((L, h), 7, dtype=torch.int32, device="cuda")
    pts = torch.full((L, 4, 3), 7.0, device="cuda")
    count = torch.full((L,), 7, dtype=torch.int32, device="cuda")
    _lib.lib()
    fn = _lib._fns["sam6d_track_points_scene"][0]
    stream = torch.cuda.current_stream().cuda_stream

    def call(L=L, H=h, W=w, margin=1, n=4, dmask=dm):
        args = [rd, depth, L, H, W, 1.0, 600.0, 600.0, 3.5, 3.5, centre, radius, margin, n, hm, dmask, cand, rows, pts, count, None]
        return fn(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args], stream)

    for kw in (dict(L=-1), dict(H=0), dict(W=0), dict(margin=-1), dict(n=0), dict(dmask=None), dict(W=49153, H=1),
               dict(L=65536, H=1, W=1), dict(H=65536, W=1)):
        assert call(**kw) == -22, kw
    torch.cuda.synchronize()
    # nothing was launched: every output and scratch buffer still holds its fill
    assert all((x == 7).all() for x in (hm, dm, cand, rows, pts, count))
    assert call(L=0, dmask=None) == 0 and call() == 0
    torch.cuda.synchronize()
    assert count.tolist() == [h * w, 0]                                     # both tracks tie everywhere: the lower one takes all


# ---- sequences ------------------------------------------------------------------------------------------------------------------
def two_copies(n=24):
    """ground truth of two copies, thin side towards the camera: A at 0.70 m turning 1 degree a frame in the image plane and
    drifting 1 mm a frame; B at 0.595 m (5 mm clear of A's front), 105 mm above, passing 8 mm a frame across in front of A
    and turning the other way.  Their centroids stay 0.15 - 0.2 m apart, inside each other's gate (about 0.17 m)."""
    Ry = tt._so3([0, 1, 0], 90)
    A = [(tt._so3([0, 0, 1], 1.0 * f) @ Ry, np.array([-0.01 + 0.001 * f, 0.0, 0.70])) for f in range(n)]
    B = [(tt._so3([0, 0, 1], -1.0 * f) @ Ry, np.array([-0.10 + 0.008 * f, -0.105, 0.595])) for f in range(n)]
    return A, B


def _frames(golden_dir, poses_per_frame, seed=0):
    rng = np.random.RandomState(seed)
    main, _, up = tt._meshes(golden_dir)
    return main, [tt.raw_depth(tt.render_depth_mm([up[0]] * len(p), p), rng) if p else np.zeros((H, W), np.uint16)
                  for p in poses_per_frame]


def run_two(main, frames, seeds, **kw):
    from sam6d_b200.track import Tracker
    det = tt._NoDetector()
    tr = Tracker(det, tt._objects_of(main), [main], max_instances=2, **kw)
    ids = [tr.start(0, R, t) for R, t in seeds]
    rgb = np.zeros((H, W, 3), np.uint8)
    return [tr(rgb, raw, K.ravel(), DEPTH_SCALE) for raw in frames], det, ids


def _err(res, slot, truth):
    R, t = res.R[slot].cpu().numpy().astype(np.float64), res.t[slot].cpu().numpy().astype(np.float64)
    if not np.isfinite(R).all():
        return np.inf, np.inf
    return io.rotation_error_deg(R, truth[0]), 1000 * np.linalg.norm(t - truth[1])


def test_two_copies_keep_their_identities(golden_dir, monkeypatch):
    from sam6d_b200 import ops, track
    A, B = two_copies()
    main, frames = _frames(golden_dir, list(zip(A, B)))
    _, clear = _frames(golden_dir, [[a] for a in A])
    hidden = [((clear[f] > 0) & (frames[f] > 0) & (frames[f] < 620)).sum() / (clear[f] > 0).sum() for f in range(len(A))]
    assert 0.2 < max(hidden) < 0.4

    def summary(res):
        e = np.array([[*_err(r, 0, a), *_err(r, 1, b)] for r, a, b in zip(res, A, B)])
        swaps = [f for f, r in enumerate(res)                             # frames where each track is nearer the other copy
                 if np.isfinite(e[f]).all() and _err(r, 0, B[f])[1] < e[f, 1] and _err(r, 1, A[f])[1] < e[f, 3]]
        return e, swaps

    res, det, ids = run_two(main, frames, [A[0], B[0]])
    e, swaps = summary(res)
    print(f"scene rule: up to {100 * max(hidden):.0f} % of A hidden; max error A {e[:, 0].max():.3f} deg {e[:, 1].max():.3f} mm, "
          f"B {e[:, 2].max():.3f} deg {e[:, 3].max():.3f} mm")
    # the shared rule on the same frames: both tracks' points through ops.track_points
    monkeypatch.setattr(track.ops, "track_points_scene", ops.track_points)
    res_s, det_s, _ = run_two(main, frames, [A[0], B[0]])
    monkeypatch.undo()
    e_s, swaps_s = summary(res_s)
    lost_s = [f for f, r in enumerate(res_s) if r.state != ["tracked", "tracked"]]
    collapsed = bool(lost_s) or bool(swaps_s) or not ((e_s[:, [0, 2]] < tt.MAX_ROT_DEG).all() and (e_s[:, [1, 3]] < tt.MAX_T_MM).all())
    mx = [float(np.max(c[np.isfinite(c)])) if np.isfinite(c).any() else float("inf") for c in e_s.T]   # over the frames tracked
    print(f"shared rule: max error A {mx[0]:.3f} deg {mx[1]:.3f} mm, B {mx[2]:.3f} deg {mx[3]:.3f} mm (while tracked); frames "
          f"with a lost or merged track {lost_s}; swaps {swaps_s}; fails the bound: {collapsed}")
    assert ids == [0, 1]
    assert all(r.state == ["tracked", "tracked"] and r.track_id.tolist() == [0, 1] for r in res), [r.state for r in res]
    assert det.calls == 1 and not swaps
    assert (e[:, [0, 2]] < tt.MAX_ROT_DEG).all() and (e[:, [1, 3]] < tt.MAX_T_MM).all(), e
    for r in res:
        assert [rec["track_id"] for rec in r.records] == [0, 1]


def test_a_copy_leaving_the_view_is_dropped(golden_dir):
    """A and B side by side at 0.7 m, about 7 px apart (inside each other's 16 px margin), A drifting towards B; B leaves the
    view at frame 4"""
    Ry = tt._so3([0, 1, 0], 90)
    A = [(Ry, np.array([-0.10 + 0.002 * f, 0.0, 0.70])) for f in range(8)]
    B = [(Ry, np.array([0.10 + 0.002 * f, 0.0, 0.70])) for f in range(8)]
    k = 4
    main, frames = _frames(golden_dir, [[a, b] if f < k else [a] for f, (a, b) in enumerate(zip(A, B))])
    res, det, ids = run_two(main, frames, [A[0], B[0]])
    print("states:", [r.state for r in res], "inliers:", [r.inliers.tolist() for r in res])
    assert all(r.state[0] == "tracked" for r in res)
    assert all(r.state == ["tracked", "tracked"] for r in res[:k])
    # B's track goes on the exit frame or the one after (a few of A's edge pixels in the margin band may keep it one more
    # frame), is never near A while it lives, and detection runs on the frame after it goes
    gone = next(f for f, r in enumerate(res) if r.state[1] == "absent")
    assert gone in (k, k + 1) and all(r.state[1] == "absent" and r.track_id[1] == -1 for r in res[gone:])
    rho = _gate(main)[1] / 1.5
    assert all(np.linalg.norm(r.t[1].cpu().numpy() - a[1]) > 0.5 * rho for r, a in zip(res[k:gone], A[k:gone]))
    assert [r.detection is not None for r in res] == [f in (0, gone + 1) for f in range(8)]
    err = np.array([_err(r, 0, a) for r, a in zip(res, A)])
    assert (err[:, 0] < tt.MAX_ROT_DEG).all() and (err[:, 1] < tt.MAX_T_MM).all(), err


def test_duplicate_track_is_merged_on_the_first_frame(golden_dir):
    A, _ = two_copies(3)
    main, frames = _frames(golden_dir, [[a] for a in A])
    off = (A[0][0], A[0][1] + np.array([0.02, 0.0, 0.0]))                  # 20 mm off, on the same copy
    res, det, ids = run_two(main, frames, [A[0], off])
    assert res[0].state == ["tracked", "absent"] and res[0].track_id.tolist() == [0, -1]
    assert res[1].detection is not None and res[1].state == ["tracked", "absent"]
    assert _err(res[0], 0, A[0])[1] < tt.MAX_T_MM


def test_two_copies_are_deterministic(golden_dir):
    A, B = two_copies(8)
    main, frames = _frames(golden_dir, list(zip(A, B)))
    a, _, _ = run_two(main, frames, [A[0], B[0]])
    b, _, _ = run_two(main, frames, [A[0], B[0]])
    drop = lambda recs: [{k: v for k, v in r.items() if k != "time"} for r in recs]          # noqa: E731
    for x, y in zip(a, b):
        assert torch.equal(x.R, y.R) and torch.equal(x.t, y.t) and np.array_equal(x.inliers, y.inliers)
        assert np.array_equal(x.track_id, y.track_id) and drop(x.records) == drop(y.records)


# ---- with the SAM6D pipeline ----------------------------------------------------------------------------------------------------
def test_detect_objects_unchanged_by_a_multi_instance_tracker(golden_dir):
    from sam6d_b200.track import Tracker
    model = tt._sam6d()
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    frame = (g["rgb"].numpy().astype(np.uint8), g["depth"].numpy().astype(np.uint16), g["cam_K"], g["depth_scale"])
    main, _, _ = tt._meshes(golden_dir)
    mesh, objs = tt._onboard(model, main)
    res0 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    tr = Tracker(model, objs, [mesh], max_instances=3, start_score=-1.0)
    first = tr(*frame)
    tr(*frame)
    res1 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    drop = lambda recs: [{k: v for k, v in r.items() if k != "time"} for r in recs]          # noqa: E731
    assert drop(res0.ism) == drop(res1.ism) and drop(res0.pem) == drop(res1.pem) and len(res0.pem) > 0
    assert torch.equal(res0.R, res1.R) and torch.equal(res0.t, res1.t)
    assert first.detection is not None and first.state[0] == "detected"
    best = int(np.argmax(first.detection.frame.pose_scores))
    assert torch.equal(first.R[0], first.detection.R[best]) and first.records[0]["track_id"] == 0
    print("multi-instance starts:", first.state, first.track_id.tolist())


def test_cli_writes_track_ids(golden_dir, tmp_path):
    import cv2
    from test_gpu_cli import _write_ply
    from sam6d_b200.cli import track_sam6d
    A, B = two_copies(3)
    main, frames = _frames(golden_dir, list(zip(A, B)))
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
                             "-1", "--max_instances", "2", "--start_score", "-1"]) == 0
    res = json.load(open(out / "sam6d_results" / "track_pem.json"))
    assert [r["frame"] for r in res] == ["000000.png", "000001.png", "000002.png"]
    keys = {"scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation", "R", "t", "track", "frames_tracked",
            "track_id"}
    n = 0
    for r in res:
        assert isinstance(r["records"], list) and len(r["records"]) <= 2
        ids = [rec["track_id"] for rec in r["records"]]
        assert len(set(ids)) == len(ids)
        for rec in r["records"]:
            n += 1
            assert set(rec) == keys and rec["category_id"] == 1 and rec["track"] in ("tracked", "detected")
            R = np.array(rec["R"])
            assert R.shape == (3, 3) and np.allclose(R @ R.T, np.eye(3), atol=1e-4) and len(rec["t"]) == 3
            assert isinstance(rec["track_id"], int) and rec["track_id"] >= 0
    assert n > 0
    print("CLI records:", [[(rec["track"], rec["track_id"]) for rec in r["records"]] for r in res])
