"""CPU: the float64 restatement of the distinct coarse hypotheses (oracle/hypotheses_oracle.py) on sets whose answer can be read
off by hand, the argument checks of Net.set_hypotheses, SAM6D and the CLIs, the pipeline's choice among hypotheses with the
device steps stubbed, and the graph cache's copy of the extra outputs."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import hypotheses_oracle as ho

COS30, D2 = ho.thresholds(30.0, 0.2)


def _rz(deg):
    a = math.radians(deg)
    return np.array([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])


def _set(Rs, ts):
    """-> Rt (1,n2,12) f32 and top (1,n2) = 0..n2-1"""
    hyp = np.concatenate([np.stack(Rs).reshape(-1, 9), np.stack(ts)], axis=1).astype(np.float32)
    return hyp[None], np.arange(len(Rs))[None]


def _picks(Rt, top, scores, K, cos_thr=COS30, d2_min=D2):
    out = []
    for fp32 in (False, True):
        R, t, sc, valid, count, pick, und = ho.pick_distinct(Rt, top, np.asarray(scores, np.float32)[None], K, cos_thr, d2_min, fp32)
        assert und[0] == 0
        out.append((pick[0].tolist(), valid[0].tolist(), int(count[0])))
    assert out[0] == out[1]                                          # fp32 order and float64 agree away from the thresholds
    return out[0]


def test_thresholds():
    from sam6d_b200 import ops
    assert ho.thresholds(30.0, 0.2) == ops.hypothesis_thresholds(30.0, 0.2)
    assert COS30 == float(np.float32(1 + math.sqrt(3))) and D2 == float(np.float32(0.04))
    assert ho.thresholds(180.0, 0.0) == (-1.0, 0.0)


def test_rotations_about_one_axis():
    """0, 10, 25, 40, 50, 90, 180 degrees about z, same t, scores falling with the index: 10 and 25 are within 30 degrees of 0,
    50 within 30 of 40; 90 and 180 are distinct from every pick"""
    Rt, top = _set([_rz(a) for a in (0, 10, 25, 40, 50, 90, 180)], [np.zeros(3)] * 7)
    scores = [7, 6, 5, 4, 3, 2, 1]
    assert _picks(Rt, top, scores, 4) == ([0, 3, 5, 6], [1, 1, 1, 1], 4)
    assert _picks(Rt, top, scores, 6) == ([0, 3, 5, 6, 0, 0], [1, 1, 1, 1, 0, 0], 4)
    assert _picks(Rt, top, scores, 2) == ([0, 3], [1, 1], 2)
    # 60 degrees apart: 10 to 50 are within 60 of 0, then 90 and 180 are picked
    c60, _ = ho.thresholds(60.0, 0.2)
    assert _picks(Rt, top, scores, 7, c60) == ([0, 5, 6, 0, 0, 0, 0], [1, 1, 1, 0, 0, 0, 0], 3)
    # the highest score decides the first pick, not the order
    assert _picks(Rt, top, [1, 2, 3, 4, 5, 6, 7], 3) == ([6, 5, 4], [1, 1, 1], 3)


def test_translations_only():
    """identity rotations at x = 0, 0.1, 0.3, 0.45 with min_dist 0.2: 0.1 is within 0.2 of 0, 0.45 within 0.2 of 0.3"""
    Rt, top = _set([np.eye(3)] * 4, [np.array([x, 0.0, 0.0]) for x in (0.0, 0.1, 0.3, 0.45)])
    assert _picks(Rt, top, [4, 3, 2, 1], 4) == ([0, 2, 0, 0], [1, 1, 0, 0], 2)
    # a rotation makes a close translation distinct
    Rt2, top2 = _set([np.eye(3), _rz(45)], [np.zeros(3), np.array([0.01, 0, 0])])
    assert _picks(Rt2, top2, [2, 1], 2) == ([0, 1], [1, 1], 2)


def test_identical_hypotheses_give_one():
    Rt, top = _set([_rz(17)] * 5, [np.array([0.1, 0.2, 0.3])] * 5)
    assert _picks(Rt, top, [1, 3, 3, 2, 0], 3) == ([1, 1, 1], [1, 0, 0], 1)        # ties: the first maximal index


def test_nan_scores():
    Rt, top = _set([_rz(a) for a in (0, 90, 180, 270)], [np.zeros(3)] * 4)
    assert _picks(Rt, top, [np.nan, 0.5, np.nan, 0.9], 4) == ([3, 1, 3, 3], [1, 1, 0, 0], 2)
    assert _picks(Rt, top, [np.nan] * 4, 3) == ([0, 0, 0], [1, 0, 0], 1)           # all NaN: hypothesis 0, as the single pick
    assert _picks(Rt, top, [-np.inf, np.nan, -np.inf, 1.0], 4) == ([3, 0, 2, 3], [1, 1, 1, 0], 3)


def test_k_equals_n2():
    Rt, top = _set([_rz(a) for a in (0, 1, 2, 3, 4)], [np.zeros(3)] * 5)
    # min_dist 0: every squared distance is >= 0, so every hypothesis is distinct: the top K by score
    assert _picks(Rt, top, [3, 5, 4, 1, 2], 5, COS30, 0.0) == ([1, 2, 0, 4, 3], [1] * 5, 5)
    assert _picks(Rt, top, [3, 5, 4, 1, 2], 5) == ([1, 1, 1, 1, 1], [1, 0, 0, 0, 0], 1)


def test_undecided_is_counted_at_the_threshold():
    """a pair exactly min_angle apart lies inside the rounding bound of its own threshold"""
    Rt, top = _set([_rz(0), _rz(30)], [np.zeros(3)] * 2)
    *_, und = ho.pick_distinct(Rt, top, np.array([[2.0, 1.0]], np.float32), 2, COS30, D2)
    assert und[0] == 1


def test_gather_of_the_picked_poses():
    rng = np.random.RandomState(0)
    Rt = rng.normal(size=(2, 9, 12)).astype(np.float32)
    top = np.stack([rng.permutation(9)[:6] for _ in range(2)])
    scores = rng.rand(2, 6).astype(np.float32)
    R, t, sc, valid, count, pick, _ = ho.pick_distinct(Rt, top, scores, 3, COS30, 0.0)
    for b in range(2):
        assert pick[b].tolist() == np.argsort(-scores[b], kind="stable")[:3].tolist()
        assert np.array_equal(R[b], Rt[b, top[b][pick[b]], :9].reshape(3, 3, 3)) and np.array_equal(sc[b], scores[b][pick[b]])


# ---- arguments -----------------------------------------------------------------------------------------------------------------
BAD = [dict(k=0), dict(k=17), dict(k=2.5), dict(k=True), dict(min_angle=0.0), dict(min_angle=-5.0), dict(min_angle=180.5),
       dict(min_angle=float("nan")), dict(min_dist=-0.1), dict(min_dist=float("inf")), dict(min_dist=float("nan"))]


def test_set_hypotheses_checks_its_arguments():
    from sam6d_b200.pem import Net
    net = Net()
    assert net.hypotheses == (1, 30.0, 0.2)
    for kw in BAD:
        with pytest.raises(ValueError):
            net.set_hypotheses(**kw)
    assert net.hypotheses == (1, 30.0, 0.2)
    assert net.set_hypotheses(16, 180.0, 0.0) is net and net.hypotheses == (16, 180.0, 0.0)
    assert net.set_hypotheses().hypotheses == (1, 30.0, 0.2)


def test_sam6d_checks_its_arguments():
    from sam6d_b200 import pipeline
    import inspect
    p = inspect.signature(pipeline.SAM6D.__init__).parameters
    assert (p["pem_hypotheses"].default, p["hyp_min_angle"].default, p["hyp_min_dist"].default) == (1, 30.0, 0.2)
    for kw in BAD:
        args = dict(pem_hypotheses=kw.get("k", 4), hyp_min_angle=kw.get("min_angle", 30.0), hyp_min_dist=kw.get("min_dist", 0.2))
        with pytest.raises(ValueError):
            pipeline.SAM6D(**args)


def test_cli_options():
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli, run_bop, run_sam6d, track_sam6d
    req = ["--cad_path", "o.ply", "--rgb_path", "r.png", "--depth_path", "d.png", "--cam_path", "c.json", "--output_dir", "out"]
    bop = ["--bop_root", "b", "--dataset_name", "ycbv", "--output_dir", "out"]
    trk = ["--cad_path", "o.ply", "--rgb_dir", "r", "--depth_dir", "d", "--cam_path", "c.json", "--output_dir", "out"]
    for parser, base in ((pem_cli.get_parser(), []), (run_sam6d.get_parser(), req), (run_bop.get_parser(), bop),
                         (track_sam6d.get_parser(), trk)):
        a = parser.parse_args(base)
        assert (a.pem_hypotheses, a.hyp_min_angle, a.hyp_min_dist) == (1, 30.0, 0.2)
        a = parser.parse_args(base + ["--pem_hypotheses", "4", "--hyp_min_angle", "45", "--hyp_min_dist", "0.1"])
        assert (a.pem_hypotheses, a.hyp_min_angle, a.hyp_min_dist) == (4, 45.0, 0.1)
    for main, base in ((pem_cli.main, []), (run_sam6d.main, req), (run_bop.main, bop), (track_sam6d.main, trk)):
        for bad in (["--pem_hypotheses", "0"], ["--pem_hypotheses", "17"], ["--hyp_min_angle", "0"], ["--hyp_min_dist", "-1"],
                    ["--verify_tau", "0"], ["--verify_tau", "inf"], ["--icp_iters", "-1"]):
            with pytest.raises(SystemExit):
                main(base + bad)


# ---- the pipeline's choice, device steps stubbed ---------------------------------------------------------------------------------
def _out(B, K, scores, valid):
    R = torch.arange(B * K * 9, dtype=torch.float32).view(B, K, 3, 3)
    t = torch.arange(B * K * 3, dtype=torch.float32).view(B, K, 3)
    s = torch.tensor(scores, dtype=torch.float32)
    return dict(hyp_R=R, hyp_t=t, hyp_pose_score=s, hyp_valid=torch.tensor(valid, dtype=torch.uint8), pred_R=R[:, 0], pred_t=t[:, 0],
                pred_pose_score=s[:, 0], hyp_index=torch.zeros(B, dtype=torch.int64))


def _stub_verify(values, log):
    def verify_out(out, meshes, obj, radii, rows, cam_K, tau):
        log.append(dict(R=out["pred_R"].clone(), obj=np.asarray(obj).copy(), mrow=np.asarray(rows.mrow).copy()))
        v = torch.tensor(values, dtype=torch.float32).reshape(-1)
        out.update(verify=v, verify_counts=torch.arange(len(v) * 6, dtype=torch.int32).view(-1, 6))
        return out
    return verify_out


def test_choice_by_pose_score_times_verify(monkeypatch):
    from sam6d_b200 import pipeline
    B, K = 2, 4
    scores = [[0.5, 0.5, 0.5, 0.5], [0.9, 0.2, 0.8, 0.8]]
    verify = [[0.07, 0.2, 1.0, 0.6], [0.5, 1.0, 0.5, 0.9]]
    log = []
    monkeypatch.setattr(pipeline, "verify_out", _stub_verify(verify, log))
    out = _out(B, K, scores, [[1, 1, 1, 1], [1, 1, 1, 0]])
    rows = SimpleNamespace(depth=None, mask=None, mrow=np.array([5, 3]))
    pipeline.finish_poses(out, torch.zeros(B, 8, 3), torch.zeros(B, 8, 3), torch.tensor([1, 0]), verify=["m0", "m1"],
                          radii=np.ones(2), rows=rows, cam_K=np.eye(3))
    # row 0: products 0.035, 0.1, 0.5, 0.3 -> 2; row 1: 0.45, 0.2, 0.4 and an invalid 0.72 -> 0
    assert out["hyp_index"].tolist() == [2, 0]
    assert torch.equal(out["pred_R"], out["hyp_R"][[0, 1], [2, 0]]) and torch.equal(out["pred_t"], out["hyp_t"][[0, 1], [2, 0]])
    assert out["pred_pose_score"].tolist() == [0.5, pytest.approx(0.9)] and out["verify"].tolist() == [1.0, 0.5]
    assert torch.equal(out["hyp_verify"], torch.tensor(verify))
    assert torch.equal(out["verify_counts"], torch.arange(48, dtype=torch.int32).view(8, 6)[[2, 4]])
    # all B K poses were verified, each against its detection's mask row and object
    assert torch.equal(log[0]["R"], out["hyp_R"].reshape(8, 3, 3))
    assert log[0]["mrow"].tolist() == [5] * 4 + [3] * 4 and log[0]["obj"].tolist() == [1] * 4 + [0] * 4
    assert "hyp_icp_R" not in out and "pem_R" not in out


def test_choice_ties_go_to_the_lowest_hypothesis(monkeypatch):
    from sam6d_b200 import pipeline
    monkeypatch.setattr(pipeline, "verify_out", _stub_verify([[0.5, 1.0, 1.0], [float("nan"), 0.0, 0.0]], []))
    out = _out(2, 3, [[1.0, 0.5, 0.5], [1.0, 1.0, 1.0]], [[1, 1, 1], [1, 1, 1]])
    pipeline.finish_poses(out, torch.zeros(2, 8, 3), torch.zeros(2, 8, 3), torch.zeros(2, dtype=torch.int64), verify=["m"],
                          radii=np.ones(1), rows=SimpleNamespace(depth=None, mask=None, mrow=np.arange(2)), cam_K=np.eye(3))
    assert out["hyp_index"].tolist() == [0, 1]                      # 0.5 = 0.5 = 0.5: the first; NaN never wins


def test_icp_refines_every_hypothesis_before_verification(monkeypatch):
    from sam6d_b200 import pipeline
    calls = []

    def icp_refine_out(out, pts, model, obj, icp, iters):
        calls.append((out["pred_R"].shape[0], pts.shape[0], obj.tolist()))
        out.update(pem_R=out["pred_R"], pem_t=out["pred_t"], pred_R=out["pred_R"] + 1000, pred_t=out["pred_t"] + 1000,
                   icp_inliers=torch.arange(out["pred_R"].shape[0], dtype=torch.int32), icp_rms=torch.zeros(out["pred_R"].shape[0]))
        return out

    log = []
    monkeypatch.setattr(pipeline, "icp_refine_out", icp_refine_out)
    monkeypatch.setattr(pipeline, "verify_out", _stub_verify([[0.1, 0.9], [0.9, 0.1]], log))
    out = _out(2, 2, [[1.0, 1.0], [1.0, 1.0]], [[1, 1], [1, 1]])
    hyp_R = out["hyp_R"].clone()
    pipeline.finish_poses(out, torch.zeros(2, 8, 3), torch.zeros(2, 8, 3), torch.tensor([0, 1]), icp=("s", "n"), icp_iters=3,
                          verify=["m0", "m1"], radii=np.ones(2), rows=SimpleNamespace(depth=None, mask=None, mrow=np.arange(2)),
                          cam_K=np.eye(3))
    assert calls == [(4, 4, [0, 0, 1, 1])]
    assert torch.equal(log[0]["R"], hyp_R.reshape(4, 3, 3) + 1000)                 # the refined poses are the verified ones
    assert out["hyp_index"].tolist() == [1, 0]
    assert torch.equal(out["pred_R"], hyp_R[[0, 1], [1, 0]] + 1000) and torch.equal(out["pem_R"], hyp_R[[0, 1], [1, 0]])
    assert out["icp_inliers"].tolist() == [1, 2] and torch.equal(out["hyp_icp_R"], hyp_R + 1000)


def test_without_verification_net_choice_stands(monkeypatch):
    from sam6d_b200 import pipeline
    calls = []
    monkeypatch.setattr(pipeline, "icp_refine_out", lambda out, pts, model, obj, icp, iters: calls.append(out["pred_R"].shape[0]))
    out = _out(2, 3, [[1.0, 2.0, 0.5], [1.0, 1.0, 1.0]], [[1, 1, 1], [1, 1, 1]])
    before = {k: v.clone() for k, v in out.items()}
    pipeline.finish_poses(out, torch.zeros(2, 8, 3), torch.zeros(2, 8, 3), torch.zeros(2, dtype=torch.int64), icp=("s", "n"),
                          icp_iters=3)
    assert calls == [2]                                                              # the reported poses only
    assert all(torch.equal(out[k], before[k]) for k in before)


def test_records_carry_the_hypothesis_only_with_several():
    from sam6d_b200 import pipeline
    out = dict(pred_pose_score=torch.tensor([0.5, 0.25]), score=torch.tensor([1.0, 1.0]), pred_R=torch.zeros(2, 3, 3),
               pred_t=torch.zeros(2, 3))
    frame = SimpleNamespace(out=out, dets=[dict(a=1), dict(a=2)])
    assert all("hypothesis" not in r for r in pipeline.pem_records(frame))
    out["hyp_index"] = torch.tensor([3, 0])
    frame = SimpleNamespace(out=out, dets=[dict(a=1), dict(a=2)])
    assert [r["hypothesis"] for r in pipeline.pem_records(frame)] == [3, 0]


# ---- the graph cache's extra outputs -------------------------------------------------------------------------------------------
def test_graph_copies_the_extra_outputs(monkeypatch):
    from sam6d_b200 import graph

    class _G:
        def replay(self):
            pass

    B, K = 2, 3
    more = (("hyp_R", (B, K, 3, 3), torch.float32), ("hyp_valid", (B, K), torch.uint8), ("hyp_index", (B,), torch.int64))
    n_more = B * K * 9 + B * K + B
    flat = torch.arange(B * graph.OUT_FLOATS + n_more, dtype=torch.float32)
    seen = []

    def fake_capture(fn, ep, n_rand, keys=()):
        seen.append(keys)
        return graph._Captured(_G(), flat, torch.zeros(B, n_rand), 1, B, more)

    sg = graph.StepGraphs()
    monkeypatch.setattr(sg, "_capture", fake_capture)
    monkeypatch.setattr(graph, "signature", lambda ep, extra=(): tuple(sorted(ep)) + tuple(extra))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    ep = dict(pts=torch.zeros(B, 8, 3))
    keys = ("hyp_R", "hyp_valid", "hyp_index")
    assert sg.run(lambda e, r: e, dict(ep), None, 6, extra=(4,), keys=keys) is None
    out = sg.run(lambda e, r: e, dict(ep), None, 6, extra=(4,), keys=keys)
    assert seen == [keys]
    o = B * graph.OUT_FLOATS
    assert out["hyp_R"].shape == (B, K, 3, 3) and torch.equal(out["hyp_R"].reshape(-1), flat[o:o + B * K * 9])
    assert out["hyp_valid"].dtype == torch.uint8 and out["hyp_valid"].reshape(-1).tolist() == list(range(o + B * K * 9, o + B * K * 10))
    assert out["hyp_index"].dtype == torch.int64 and out["hyp_index"].tolist() == [o + B * K * 10, o + B * K * 10 + 1]
    # the hyp_* results of an earlier call are not part of the next call's signature
    assert graph._MORE_NAMES == frozenset(("hyp_init_R", "hyp_init_t", "hyp_R", "hyp_t", "hyp_pose_score", "hyp_valid", "hyp_index"))
    from sam6d_b200.pem import HYP_KEYS
    assert frozenset(HYP_KEYS) == graph._MORE_NAMES
