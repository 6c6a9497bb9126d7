"""GPU: several coarse hypotheses per proposal (Net.set_hypotheses, ops.coarse_pick_distinct, pipeline.finish_poses).

- K = 1 is the reference's forward, launch by launch and replayed as a graph, with no hyp_* output.
- The pick kernel against oracle/hypotheses_oracle.py at the bench shape and on constructed sets.  The kernel's fp32 order is
  restated exactly by the oracle's fp32 mode, which must match on every row; the float64 oracle must match on every row without
  an "undecided" comparison (one whose outcome can change inside the fp32 rounding bound of the trace or the squared distance:
  gamma_9 sum |R_i[e] R_j[e]|, gamma_5 d2), whose count is printed.
- Each of the K fine passes is the fine stage from that hypothesis (forward(init_pose=...)), bit for bit, and the reported pose
  is the first valid pass with the largest pose score.
- Graph replay at K = 4, and K switched between calls.
- Selection by verification on the rendered ranking scene of test_gpu_verify.py, with and without ICP, and end to end through
  SAM6D and run_sam6d."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import hypotheses_oracle as ho
from oracle import icp_oracle as io
from oracle import pem_oracle as po

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_icp import _rot, _sam6d, _scene_meshes, hull_mesh_mm             # noqa: E402,F401
from test_gpu_verify import K as CAM_K, _radius, _scene                        # noqa: E402

pytestmark = pytest.mark.gpu

KEYS = ("init_R", "init_t", "pred_R", "pred_t", "pred_pose_score")
HYP = ("hyp_init_R", "hyp_init_t", "hyp_R", "hyp_t", "hyp_pose_score", "hyp_valid", "hyp_index")


def _net(precision):
    from sam6d_b200.pem import Net
    net = Net().cuda().eval()
    net.load_state_dict(po.make_state_dict(seed=1), strict=True)
    return net.set_precision(precision)


def _inputs(B, seed):
    inp = po.make_inputs(B=B, n=2048, seed=seed)
    return {k: inp[k].cuda() for k in ("pts", "dense_fm", "dense_po", "dense_fo", "model")}


def _rand(B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(B, po.N_PROPOSAL1 * 3, device="cuda", generator=g)


def _same(a, b, keys, label):
    for k in keys:
        assert torch.equal(a[k], b[k]), (label, k)


# ---- 1. K = 1 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_one_hypothesis_is_the_reference_forward(precision):
    B = 4
    dev, rand = _inputs(B, 3), _rand(B, 5)
    plain = _net(precision)
    want = {k: v.clone() for k, v in plain(dict(dev), rand=rand).items() if k in KEYS}
    net = _net(precision).set_hypotheses(4).set_hypotheses(1)
    out = net(dict(dev), rand=rand)
    _same(out, want, KEYS, "launch by launch")
    assert not any(k in out for k in HYP)
    net.enable_graphs()
    for i in range(3):                                   # sighting, capture + replay, replay
        out = net(dict(dev), rand=rand)
        _same(out, want, KEYS, f"graph call {i}")
        assert not any(k in out for k in HYP)
    assert net._graphs.replays == 2


# ---- 2. the pick kernel against the oracle ------------------------------------------------------------------------------------
def _coarse_arrays(monkeypatch, net, dev, rand):
    """the Rt, top and scores coarse_select sees in one forward, and its R, t"""
    from sam6d_b200 import ops
    rec = {}
    orig = ops.coarse_select

    def spy(Rt, top, pts1, w1, model):
        R, t, s = orig(Rt, top, pts1, w1, model)
        rec.update(Rt=Rt, top=top, scores=s, R=R, t=t)
        return R, t, s

    monkeypatch.setattr(ops, "coarse_select", spy)
    out = net(dict(dev), rand=rand)
    monkeypatch.setattr(ops, "coarse_select", orig)
    return rec, out


def _check_kernel(ops, Rt, top, scores, K, min_angle, min_dist, label):
    """the kernel's picks against both oracle modes -> number of undecided comparisons"""
    R, t, sc, valid, count = ops.coarse_pick_distinct(Rt, top, scores, K, min_angle, min_dist)
    cos_thr, d2_min = ho.thresholds(min_angle, min_dist)
    a = [x.cpu().numpy() for x in (Rt, top, scores)]
    got = [x.cpu().numpy() for x in (R, t, sc, valid, count)]
    R32, t32, s32, v32, c32, _, _ = ho.pick_distinct(*a, K, cos_thr, d2_min, fp32=True)
    assert np.array_equal(got[3], v32) and np.array_equal(got[4], c32), label
    assert np.array_equal(got[0], R32.astype(np.float32)) and np.array_equal(got[1], t32.astype(np.float32)), label
    assert np.array_equal(got[2], s32.astype(np.float32), equal_nan=True), label
    R64, t64, s64, v64, c64, _, und = ho.pick_distinct(*a, K, cos_thr, d2_min)
    sure = und == 0
    assert np.array_equal(got[3][sure], v64[sure]) and np.array_equal(got[4][sure], c64[sure]), label
    assert np.array_equal(got[0][sure], R64[sure].astype(np.float32)) and np.array_equal(got[1][sure], t64[sure].astype(np.float32))
    # slots past the count are copies of slot 0
    for b in range(len(got[4])):
        n = got[4][b]
        assert (got[0][b, n:] == got[0][b, :1]).all() and (got[1][b, n:] == got[1][b, :1]).all() and not got[3][b, n:].any()
    print(f"{label}: counts {np.bincount(got[4], minlength=K + 1).tolist()}, {int(und.sum())} undecided comparisons in "
          f"{int((und > 0).sum())} rows")
    return R, t


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_pick_kernel_against_the_oracle(monkeypatch, precision):
    from sam6d_b200 import ops
    B = 32
    net = _net(precision)
    dev, rand = _inputs(B, 100), _rand(B, 1)
    rec, out = _coarse_arrays(monkeypatch, net, dev, rand)
    assert torch.equal(rec["R"], out["init_R"]) and torch.equal(rec["t"], out["init_t"])
    for K in (4, 8):
        for min_angle, min_dist in ((30.0, 0.2), (90.0, 0.5), (5.0, 0.02)):
            R, t = _check_kernel(ops, rec["Rt"], rec["top"], rec["scores"], K, min_angle, min_dist,
                                 f"{precision} K={K} {min_angle} deg {min_dist}")
            assert torch.equal(R[:, 0], out["init_R"]) and torch.equal(t[:, 0], out["init_t"])      # slot 0 is init_R, init_t


def _dev_set(Rs, ts, scores):
    hyp = np.concatenate([np.stack(Rs).reshape(-1, 9), np.stack(ts)], axis=1).astype(np.float32)
    n2 = len(hyp)
    perm = np.random.RandomState(n2).permutation(n2 + 3)[:n2]                      # top indexes a larger Rt
    Rt = np.random.RandomState(1).normal(size=(1, n2 + 3, 12)).astype(np.float32)
    Rt[0, perm] = hyp
    return (torch.from_numpy(Rt).cuda(), torch.from_numpy(perm[None].astype(np.int32)).cuda(),
            torch.from_numpy(np.asarray(scores, np.float32)[None]).cuda())


def _rz(deg):
    return io.so3_exp(np.radians(deg) * np.array([0.0, 0.0, 1.0]))


def test_pick_kernel_constructed_sets():
    from sam6d_b200 import ops
    z = [np.zeros(3)]
    cases = {
        "rotations about z": (_dev_set([_rz(a) for a in (0, 10, 25, 40, 50, 90, 180)], z * 7, [7, 6, 5, 4, 3, 2, 1]), 6, 30.0, 0.2,
                              [1, 1, 1, 1, 0, 0]),
        "translations": (_dev_set([np.eye(3)] * 4, [np.array([x, 0, 0]) for x in (0, 0.1, 0.3, 0.45)], [4, 3, 2, 1]), 4, 30.0, 0.2,
                         [1, 1, 0, 0]),
        "identical": (_dev_set([_rz(17)] * 5, [np.array([0.1, 0.2, 0.3])] * 5, [1, 3, 3, 2, 0]), 3, 30.0, 0.2, [1, 0, 0]),
        "NaN scores": (_dev_set([_rz(a) for a in (0, 90, 180, 270)], z * 4, [np.nan, 0.5, np.nan, 0.9]), 4, 30.0, 0.2, [1, 1, 0, 0]),
        "all NaN": (_dev_set([_rz(a) for a in (0, 90, 180, 270)], z * 4, [np.nan] * 4), 3, 30.0, 0.2, [1, 0, 0]),
        "K = n2": (_dev_set([_rz(a) for a in (0, 1, 2, 3, 4)], z * 5, [3, 5, 4, 1, 2]), 5, 30.0, 0.0, [1] * 5),
    }
    for label, ((Rt, top, scores), K, ang, dist, valid) in cases.items():
        _check_kernel(ops, Rt, top, scores, K, ang, dist, label)
        assert ops.coarse_pick_distinct(Rt, top, scores, K, ang, dist)[3][0].tolist() == valid, label
    # a large n2 (every CTA thread owns several hypotheses) and a batch of rows
    rng = np.random.RandomState(3)
    B, n1, n2 = 5, 3000, 2048
    Rt = np.zeros((B, n1, 12), np.float32)
    Rt[..., :9] = np.stack([_rot(rng) for _ in range(B * n1)]).reshape(B, n1, 9)
    Rt[..., 9:] = rng.normal(scale=0.3, size=(B, n1, 3))
    top = np.stack([rng.permutation(n1)[:n2] for _ in range(B)]).astype(np.int32)
    scores = rng.rand(B, n2).astype(np.float32)
    scores[1, ::7] = np.nan
    scores[2] = 0.5                                                                  # all tied: index order
    args = [torch.from_numpy(x).cuda() for x in (Rt, top, scores)]
    for K in (1, 8, 16):
        _check_kernel(ops, *args, K, 30.0, 0.2, f"n2 = {n2}, K = {K}")


def test_pick_kernel_invalid_arguments():
    from sam6d_b200 import _lib, ops
    B, n1, n2, K = 2, 10, 6, 3
    Rt = torch.randn(B, n1, 12, device="cuda")
    top = torch.arange(n2, dtype=torch.int32, device="cuda").repeat(B, 1).contiguous()
    sc = torch.rand(B, n2, device="cuda")
    outs = [torch.full((B, K, 3, 3), -7.0, device="cuda"), torch.full((B, K, 3), -7.0, device="cuda"), torch.full((B, K), -7.0, device="cuda"),
            torch.full((B, K), 9, dtype=torch.uint8, device="cuda"), torch.full((B,), -7, dtype=torch.int32, device="cuda")]
    before = [o.clone() for o in outs]

    def run(k=K, n2_=n2, cos_thr=2.0, d2=0.04, n1_=n1, B_=B, rt=Rt):
        _lib.call("sam6d_coarse_pick_distinct", rt, top, sc, B_, n1_, n2_, k, cos_thr, d2, *outs)

    for kw in (dict(k=0), dict(k=-1), dict(k=n2 + 1), dict(n2_=2049, k=3), dict(n2_=0), dict(cos_thr=float("nan")),
               dict(cos_thr=float("inf")), dict(d2=float("nan")), dict(d2=float("inf")), dict(d2=-float("inf")), dict(n1_=0),
               dict(B_=-1), dict(rt=None)):
        with pytest.raises(_lib.Sam6dError, match="invalid argument"):
            run(**kw)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, before))
    for kw in (dict(K=0), dict(K=n2 + 1), dict(min_angle=float("nan")), dict(min_dist=float("inf"))):
        a = {**dict(K=K, min_angle=30.0, min_dist=0.2), **kw}
        with pytest.raises(_lib.Sam6dError, match="invalid argument"):
            ops.coarse_pick_distinct(Rt, top, sc, a["K"], a["min_angle"], a["min_dist"])
    run(B_=0)                                                                        # nothing to do
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, before))


# ---- 3 and 4. the fine passes and the choice ------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_each_pass_is_the_fine_stage_and_the_best_is_reported(precision):
    B, K = 16, 4
    dev, rand = _inputs(B, 7), _rand(B, 8)
    net = _net(precision)
    one = {k: v.clone() for k, v in net(dict(dev), rand=rand).items() if k in KEYS}
    out = net.set_hypotheses(K)(dict(dev), rand=rand)
    assert out["hyp_R"].shape == (B, K, 3, 3) and out["hyp_valid"].dtype == torch.uint8 and out["hyp_index"].shape == (B,)
    assert torch.equal(out["init_R"], one["init_R"]) and torch.equal(out["init_t"], one["init_t"])
    assert torch.equal(out["hyp_init_R"][:, 0], one["init_R"]) and torch.equal(out["hyp_init_t"][:, 0], one["init_t"])
    # pass 0 starts where the single-hypothesis forward starts
    assert torch.equal(out["hyp_R"][:, 0], one["pred_R"]) and torch.equal(out["hyp_pose_score"][:, 0], one["pred_pose_score"])
    for k in range(K):
        ref = net(dict(dev), rand=rand, init_pose=(out["hyp_init_R"][:, k], out["hyp_init_t"][:, k]))
        assert "hyp_R" not in ref
        assert torch.equal(out["hyp_R"][:, k], ref["pred_R"]) and torch.equal(out["hyp_t"][:, k], ref["pred_t"]), k
        assert torch.equal(out["hyp_pose_score"][:, k], ref["pred_pose_score"]), k
    s, v = out["hyp_pose_score"].cpu().numpy(), out["hyp_valid"].cpu().numpy()
    idx = out["hyp_index"].cpu().numpy()
    for b in range(B):
        cand = np.where(v[b] == 1, s[b], -np.inf)
        assert idx[b] == int(np.flatnonzero(cand == cand.max())[0]) and v[b, idx[b]] == 1
    rows = torch.arange(B, device="cuda")
    hi = out["hyp_index"]
    assert torch.equal(out["pred_R"], out["hyp_R"][rows, hi]) and torch.equal(out["pred_t"], out["hyp_t"][rows, hi])
    assert torch.equal(out["pred_pose_score"], out["hyp_pose_score"][rows, hi])
    print(f"{precision}: valid per proposal {v.sum(axis=1).tolist()}, chosen {idx.tolist()}")


# ---- 5. graph replay --------------------------------------------------------------------------------------------------------------
def test_graph_replay_with_hypotheses():
    from sam6d_b200 import _lib
    B = 8
    dev, rands = _inputs(B, 11), [_rand(B, 12), _rand(B, 13)]
    net = _net("bf16").set_hypotheses(4)
    want = [{k: v.clone() for k, v in net(dict(dev), rand=r).items() if k in KEYS + HYP} for r in rands]
    l0 = _lib.launch_count()
    net(dict(dev), rand=rands[0])
    per_step = _lib.launch_count() - l0
    net.enable_graphs()
    sg = net._graphs
    for i in range(4):
        l0 = _lib.launch_count()
        out = net(dict(dev), rand=rands[i % 2])
        assert _lib.launch_count() - l0 == per_step
        for k in KEYS + HYP:
            assert out[k].dtype == want[i % 2][k].dtype and torch.equal(out[k], want[i % 2][k]), (i, k)
    assert sg.captures == 1 and sg.replays == 3
    ep = dict(dev)
    net(ep, rand=rands[0])                                  # a dict that carries hyp_* results keeps its signature
    net(ep, rand=rands[0])
    assert sg.captures == 1 and sg.replays == 5
    # another K is another signature: seen launch by launch first, never the K = 4 graph
    net.set_hypotheses(2)
    out = net(dict(dev), rand=rands[0])
    assert sg.replays == 5 and out["hyp_R"].shape == (B, 2, 3, 3)
    out = net(dict(dev), rand=rands[0])
    assert sg.replays == 6 and sg.captures == 2 and out["hyp_R"].shape == (B, 2, 3, 3)
    net.disable_graphs()
    eager = net(dict(dev), rand=rands[0])
    for k in KEYS + HYP:
        assert torch.equal(out[k], eager[k]), k
    net.enable_graphs().set_hypotheses(1)
    for _ in range(2):
        out = net(dict(dev), rand=rands[0])
        assert not any(k in out for k in HYP)
    net.set_hypotheses(4, 45.0)                              # other thresholds: another signature too
    out = net(dict(dev), rand=rands[0])
    assert net._graphs.replays == 1 and out["hyp_R"].shape == (B, 4, 3, 3)


# ---- 6. selection by verification ----------------------------------------------------------------------------------------------
def _observed(depth, mask, n=2048):
    ys, xs = torch.nonzero((mask > 0) & (depth > 0), as_tuple=True)
    sel = torch.linspace(0, len(ys) - 1, n, device="cuda").long()
    ys, xs = ys[sel], xs[sel]
    z = depth[ys, xs]
    fx, fy, cx, cy = (float(CAM_K[0, 0]), float(CAM_K[1, 1]), float(CAM_K[0, 2]), float(CAM_K[1, 2]))
    return torch.stack([(xs.float() - cx) * z / fx, (ys.float() - cy) * z / fy, z], dim=1)[None].contiguous()


def test_selection_by_verification(golden_dir):
    from sam6d_b200 import ops, pipeline
    meshes, ((R0, t0), _), depth, masks, hidden = _scene(11)
    ray = t0 / np.linalg.norm(t0)
    axis = np.random.RandomState(12).normal(size=3)
    poses = [(np.diag([-1.0, -1.0, 1.0]) @ R0, t0), (R0, t0 + 0.010 * ray), (R0, t0),
             (R0 @ io.so3_exp(np.radians(15) * axis / np.linalg.norm(axis)), t0)]
    names = ["flipped", "10 mm behind", "true", "15 deg rotated"]
    hyp_R = torch.from_numpy(np.stack([p[0] for p in poses]).astype(np.float32))[None].cuda()
    hyp_t = torch.from_numpy(np.stack([p[1] for p in poses]).astype(np.float32))[None].cuda()
    rows = SimpleNamespace(depth=depth, mask=masks, mrow=np.array([0]))
    radii = np.array([_radius(meshes, 0), _radius(meshes, 1)])

    def fresh():
        s = torch.full((1, 4), 0.8, device="cuda")
        return dict(hyp_R=hyp_R.clone(), hyp_t=hyp_t.clone(), hyp_pose_score=s, hyp_valid=torch.ones(1, 4, dtype=torch.uint8, device="cuda"),
                    pred_R=hyp_R[:, 0].clone(), pred_t=hyp_t[:, 0].clone(), pred_pose_score=s[:, 0].clone(),
                    hyp_index=torch.zeros(1, dtype=torch.int64, device="cuda"))

    obj = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = pipeline.finish_poses(fresh(), torch.zeros(1, 8, 3, device="cuda"), torch.zeros(1, 8, 3, device="cuda"), obj,
                                verify=meshes, radii=radii, rows=rows, cam_K=CAM_K, verify_tau=0.1)
    v = out["hyp_verify"][0].cpu().numpy()
    print("verify per hypothesis:", dict(zip(names, v.round(4).tolist())))
    assert int(out["hyp_index"][0]) == 2
    assert torch.equal(out["pred_R"], hyp_R[:, 2]) and torch.equal(out["pred_t"], hyp_t[:, 2])
    counts, want = ops.verify_poses(hyp_R[0], hyp_t[0], [0] * 4, meshes, depth, masks, [0] * 4, CAM_K, 0.1 * radii[0])
    assert torch.equal(out["hyp_verify"][0], want) and torch.equal(out["verify_counts"], counts[2:3])
    assert float(out["verify"][0]) == float(want[2]) and float(out["pred_pose_score"][0]) == pytest.approx(0.8)
    # with ICP every hypothesis is refined first, and the refined poses are the verified ones
    v0, f0 = hull_mesh_mm(golden_dir)
    samples, normals = pipeline.icp_model(v0, f0)
    icp = pipeline.icp_tensors(samples, normals, "cuda")
    pts = _observed(depth, masks[0])
    model = icp[0][:1].contiguous()
    out = pipeline.finish_poses(fresh(), pts, model, obj, icp=icp, icp_iters=10, verify=meshes, radii=radii, rows=rows, cam_K=CAM_K,
                                verify_tau=0.1)
    R_icp, t_icp, inl, _, _ = ops.icp_refine(hyp_R[0], hyp_t[0], pts.expand(4, -1, -1).contiguous(), icp[0], icp[1],
                                             torch.zeros(4, dtype=torch.int32, device="cuda"),
                                             model.norm(dim=2).amax(dim=1).expand(4).contiguous(), 10)
    assert torch.equal(out["hyp_icp_R"][0], R_icp) and torch.equal(out["hyp_icp_t"][0], t_icp)
    _, want = ops.verify_poses(R_icp, t_icp, [0] * 4, meshes, depth, masks, [0] * 4, CAM_K, 0.1 * radii[0])
    assert torch.equal(out["hyp_verify"][0], want)
    k = int(out["hyp_index"][0])
    prod = (0.8 * want).cpu().numpy()
    assert k == int(np.argmax(prod)) and prod[k] >= prod[2]
    assert torch.equal(out["pred_R"][0], R_icp[k]) and torch.equal(out["pem_R"][0], hyp_R[0, k]) and int(out["icp_inliers"][0]) == int(inl[k])
    print("verify after ICP:", dict(zip(names, want.cpu().numpy().round(4).tolist())), "chosen", names[k])


# ---- 7. end to end ----------------------------------------------------------------------------------------------------------------
def _check_records(res, res1, icp):
    out = res.frame.out
    P = len(res.pem)
    assert P == len(res1.pem) > 0
    drop = ("time", "score", "R", "t", "verify", "hypothesis")
    strip = lambda recs: [{k: v for k, v in r.items() if k not in drop} for r in recs]            # noqa: E731
    assert strip(res.pem) == strip(res1.pem)
    assert [{k: v for k, v in r.items() if k != "time"} for r in res.ism] == [{k: v for k, v in r.items() if k != "time"} for r in res1.ism]
    assert torch.equal(res.boxes, res1.boxes) and torch.equal(res.scores, res1.scores)
    hR = out["hyp_icp_R"] if icp else out["hyp_R"]
    ht = out["hyp_icp_t"] if icp else out["hyp_t"]
    idx = out["hyp_index"].cpu().numpy()
    valid = out["hyp_valid"].cpu().numpy()
    prod = (out["hyp_pose_score"] * out["hyp_verify"]).cpu().numpy()
    for i, r in enumerate(res.pem):
        k = r["hypothesis"]
        assert k == idx[i] and valid[i, k] == 1
        assert torch.equal(out["pred_R"][i], hR[i, k]) and torch.equal(out["pred_t"][i], ht[i, k])
        assert np.allclose(np.asarray(r["R"]), hR[i, k].cpu().numpy()) and np.allclose(np.asarray(r["t"]), ht[i, k].cpu().numpy() * 1000)
        cand = np.where(valid[i] == 1, prod[i], -np.inf)
        assert k == int(np.flatnonzero(cand == cand.max())[0])
        assert r["score"] == float((out["pred_pose_score"][i] * out["score"][i] * out["verify"][i]).cpu())
        assert prod[i, k] == cand.max()                                                  # the maximal pose score x verify
    print(f"{P} poses, hypotheses {idx.tolist()}, valid {valid.sum(axis=1).tolist()}")


def test_sam6d_end_to_end(golden_dir):
    model = _sam6d()
    meshes, frame = _scene_meshes(golden_dir)
    try:
        model.verify = True
        objs = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
        one = model.onboard(meshes[0], template_size=192, rng=np.random.RandomState(0))
        for icp_iters in (0, 10):
            model.icp_iters = icp_iters
            if icp_iters:
                objs = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
            model.pem.set_hypotheses(1)
            res1 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
            assert all("hypothesis" not in r for r in res1.pem)
            model.pem.set_hypotheses(4)
            res4 = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
            _check_records(res4, res1, icp_iters > 0)
        model.icp_iters = 0
        model.pem.set_hypotheses(1)
        s1 = model(*frame, one, rng=np.random.RandomState(5))
        model.pem.set_hypotheses(4)
        s4 = model(*frame, one, rng=np.random.RandomState(5))
        _check_records(s4, s1, False)
    finally:
        model.verify, model.icp_iters = False, 0
        model.pem.set_hypotheses(1)


def test_run_sam6d_with_hypotheses(golden_dir, tmp_path):
    import json
    import cv2
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
    args = ["--output_dir", str(out), "--cad_path", cad, "--rgb_path", str(tmp_path / "rgb.png"), "--depth_path", str(tmp_path / "depth.png"),
            "--cam_path", str(tmp_path / "camera.json"), "--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1",
            "--det_score_thresh", "-1", "--template_size", "192", "--verify"]
    with pytest.raises(SystemExit):
        run_sam6d.main(args + ["--pem_hypotheses", "0"])
    assert run_sam6d.main(args + ["--pem_hypotheses", "4"]) == 0
    r = out / "sam6d_results"
    pem = json.load(open(r / "detection_pem.json"))
    print(f"run_sam6d --pem_hypotheses 4 --verify: {len(pem)} poses, hypotheses {[x['hypothesis'] for x in pem]}")
    assert pem and all(0 <= x["hypothesis"] < 4 and 0.0 <= x["verify"] <= 1.0 for x in pem) and (r / "vis_pem.png").exists()
    assert (r / "detection_ism.json").exists()
