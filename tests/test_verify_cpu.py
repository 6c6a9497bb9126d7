"""CPU: the float64 restatement of the pose verification (oracle/verify_oracle.py) on hand-built frames, its fp32 rounding
bound, the score, argument validation, CLI parsing and the defaults that leave verification off."""
import inspect

import numpy as np
import pytest
import torch

from oracle import verify_oracle as vo

TAU = 0.25
EPS = 2.0 ** -20


def hand_frame():
    """one row of pixels per case, rscale 1 and tau 0.25, every value dyadic (exact in fp32, so the kernel's classes equal
    these): (rendered dr, observed do, mask) and the classes each pixel must have"""
    cases = [
        # dr, do, mask, expected classes
        (0.0, 1.0, 1, {"mask"}),                                        # no silhouette, in the mask
        (0.0, 0.0, 0, set()),                                           # nothing
        (1.0, 1.25, 1, {"sil", "fit", "mask", "mask_fit"}),             # e = +tau: fit (upper boundary)
        (1.0, 0.75, 0, {"sil", "fit"}),                                 # e = -tau: fit (lower boundary)
        (1.0, 1.25 + EPS, 1, {"sil", "viol", "mask"}),                  # just above +tau: violation
        (1.0, 0.75 - EPS, 1, {"sil", "occ", "mask"}),                   # just below -tau: occluded
        (1.0, 1.5, 0, {"sil", "viol"}),                                 # the sensor sees behind the surface
        (1.0, 0.5, 1, {"sil", "occ", "mask"}),                          # something in front
        (1.0, 0.0, 1, {"sil", "mask"}),                                 # invalid observed depth: silhouette only
        (1.0, 1.0, 1, {"sil", "fit", "mask", "mask_fit"}),              # exact agreement
        (0.5, 0.5 + TAU - EPS, 0, {"sil", "fit"}),                      # just inside +tau
    ]
    rd = np.array([[c[0] for c in cases]], np.float32)
    do = np.array([c[1] for c in cases], np.float32)[None]
    mask = np.array([[c[2] for c in cases]], np.uint8)
    return rd[None], do, mask[None], cases


def test_oracle_classes_on_a_hand_built_frame():
    rd, do, mask, cases = hand_frame()
    c = vo.classes(rd, do, mask, [0], [TAU], 1.0)
    for i, (_, _, _, want) in enumerate(cases):
        got = {k for k in ("sil", "occ", "fit", "viol", "mask", "mask_fit") if c[k][0, 0, i]}
        assert got == want, (i, got, want)
    n = vo.counts(rd, do, mask, [0], [TAU], 1.0)
    assert n.tolist() == [[9, 2, 4, 2, 7, 2]]
    fit_frac, cover, v = vo.score(n)
    assert fit_frac[0] == 4 / 6 and cover[0] == 2 / 7 and v[0] == (4 / 6) * (2 / 7)
    # only the two pixels exactly at +-tau lie within the fp32 bound u (|e| + 2 |dr|) ~ 2^-23 of a boundary; the cases 2^-20
    # away are decided
    assert np.flatnonzero(vo.undecided(rd, do, [TAU], 1.0)[0, 0]).tolist() == [2, 3]


def test_oracle_zero_denominators():
    H, W = 3, 4
    do = np.full((H, W), 1.0, np.float32)
    rd = np.zeros((4, H, W), np.float32)
    rd[1] = 1.0                                           # fits everywhere
    rd[2] = 2.0                                           # behind the observed surface everywhere: all occluded
    rd[3, 0, 0] = 1.0
    mask = np.zeros((2, H, W), np.uint8)
    mask[1, :, :2] = 1
    mrow = [1, 0, 1, 1]                                   # hypothesis 1 reads the empty mask row
    n = vo.counts(rd, do, mask, mrow, [TAU] * 4, 1.0)
    fit_frac, cover, v = vo.score(n)
    assert n[0].tolist() == [0, 0, 0, 0, 6, 0] and fit_frac[0] == 0 and cover[0] == 0 and v[0] == 0      # no silhouette
    assert n[1].tolist() == [12, 0, 12, 0, 0, 0] and fit_frac[1] == 1 and cover[1] == 0 and v[1] == 0    # empty mask
    assert n[2].tolist() == [12, 12, 0, 0, 6, 0] and fit_frac[2] == 0 and v[2] == 0                     # fully occluded
    assert n[3].tolist() == [1, 0, 1, 0, 6, 1] and fit_frac[3] == 1 and cover[3] == 1 / 6
    assert np.isfinite(v).all()


def _fp32_kernel_classes(rd, do, tau, rscale):
    """the kernel's arithmetic in numpy fp32 (IEEE, rounded to nearest, no contraction)"""
    dr = rd.astype(np.float32) * np.float32(rscale)
    e = do.astype(np.float32)[None] - dr
    t = np.float32(tau)
    seen = (dr > 0) & (do[None] > 0)
    return seen & (e < -t), seen & (np.abs(e) <= t), seen & (e > t)


def test_fp32_classes_differ_from_the_oracle_only_on_undecided_pixels():
    """random depths in mm at a tolerance of 5 mm, many of them within a few ulps of the boundaries"""
    rng = np.random.RandomState(0)
    rscale = float(np.float32(1e-3))
    tau = float(np.float32(0.005))
    rd = rng.uniform(300.0, 900.0, size=(3, 64, 64)).astype(np.float32)
    do = (rd[0].astype(np.float64) * rscale + rng.choice([-tau, tau], size=(64, 64)) * (1 + rng.randint(-4, 5, size=(64, 64)) * 2.0 ** -23))
    do = do.astype(np.float32)
    c = vo.classes(rd, do, np.zeros((1, 64, 64), np.uint8), [0, 0, 0], [tau] * 3, rscale)
    und = vo.undecided(rd, do, [tau] * 3, rscale)
    occ, fit, viol = _fp32_kernel_classes(rd, do, tau, rscale)
    for name, k in (("occ", occ), ("fit", fit), ("viol", viol)):
        diff = k != c[name]
        assert not (diff & ~und).any(), name
    assert und[0].sum() > 0                     # the bound is exercised
    assert und[1:].sum() < und[0].sum()


def test_verify_score_matches_the_oracle():
    from sam6d_b200 import ops
    rng = np.random.RandomState(1)
    n = rng.randint(0, 5000, size=(50, 6))
    n[:5, 2:4] = 0                                        # 0 / 0 fit fraction
    n[5:10, 4] = 0                                        # 0 / 0 cover
    n[:, 5] = np.minimum(n[:, 5], n[:, 4])
    got = ops.verify_score(torch.from_numpy(n.astype(np.int32))).numpy()
    want = vo.score(n)[2]
    assert got.dtype == np.float32 and np.all(np.abs(got - want) <= 3 * 2.0 ** -24 * want + 1e-30)
    assert (got[:10] == 0).all()


def test_verify_rows_validation():
    from sam6d_b200 import ops
    m, t = ops.verify_rows(np.array([0, 2, 1]), 0.01, 3, 3)
    assert m.dtype == np.int32 and t.dtype == np.float32 and t.tolist() == [np.float32(0.01)] * 3
    for mrow, tau in (([0, 3, 1], 0.01), ([-1, 0, 0], 0.01), ([0, 0, 0], 0.0), ([0, 0, 0], -1.0), ([0, 0, 0], float("nan")),
                      ([0, 0, 0], float("inf")), ([0, 0, 0], 1e-50), ([0, 0, 0], [0.1, 0.1, 0.0]), ([0, 0], 0.1),
                      ([0.0, 1.0, 2.0], 0.1)):
        with pytest.raises(ValueError):
            ops.verify_rows(np.asarray(mrow), tau, 3, 3)
    assert ops.verify_rows(np.zeros(0, np.int64), np.zeros(0), 0, 1)[0].shape == (0,)


def test_sam6d_rejects_a_bad_tolerance_and_a_mesh_without_faces():
    from sam6d_b200 import pipeline
    for tau in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="verify_tau"):
            pipeline.SAM6D(verify=True, verify_tau=tau)
    v = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError, match="faces"):
        pipeline.verify_mesh(v, np.zeros((0, 3), np.int64), "cpu")


def test_defaults_leave_verification_off():
    from sam6d_b200 import pipeline
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli, run_bop, run_sam6d, track_sam6d
    p = inspect.signature(pipeline.SAM6D.__init__).parameters
    assert p["verify"].default is False and p["verify_tau"].default == 0.1
    # verification, ICP and symmetries are off and hold nothing unless asked for
    assert all(x is None for x in pipeline.PoseInputs()) and pipeline.PoseInputs._fields == ("icp", "meshes", "radii", "symmetries")
    assert inspect.signature(pipeline.pem_frame).parameters["pose"].default == pipeline.PoseInputs()
    assert pipeline.Onboarded.__dataclass_fields__["pose_inputs"].default == pipeline.PoseInputs()
    assert pipeline.ObjectSet.__dataclass_fields__["pose_inputs"].default == pipeline.PoseInputs()
    assert pipeline.build_pose_inputs([None], np.ones((1, 4, 3)), "cpu") == pipeline.PoseInputs()
    req = ["--cad_path", "o.ply", "--rgb_path", "r.png", "--depth_path", "d.png", "--cam_path", "c.json", "--output_dir", "out"]
    bop = ["--bop_root", "b", "--dataset_name", "ycbv", "--output_dir", "out"]
    trk = ["--cad_path", "o.ply", "--rgb_dir", "r", "--depth_dir", "d", "--cam_path", "c.json", "--output_dir", "out"]
    for parser, base in ((pem_cli.get_parser(), []), (run_sam6d.get_parser(), req), (run_bop.get_parser(), bop),
                         (track_sam6d.get_parser(), trk)):
        a = parser.parse_args(base)
        assert a.verify is False and a.verify_tau == 0.1
        a = parser.parse_args(base + ["--verify", "--verify_tau", "0.05"])
        assert a.verify is True and a.verify_tau == 0.05


def _frame(verify):
    from types import SimpleNamespace
    out = dict(pred_pose_score=torch.tensor([0.5, 0.9, 0.3]), score=torch.tensor([0.7, 0.3, 0.6]),
               pred_R=torch.eye(3).repeat(3, 1, 1), pred_t=torch.tensor([[0.01, 0.02, 0.5]] * 3))
    if verify:
        out.update(verify=torch.tensor([0.25, 0.0, 0.8]), verify_counts=torch.zeros(3, 6, dtype=torch.int32))
    dets = [dict(scene_id=0, image_id=0, category_id=1, bbox=[0, 0, 1, 1], score=float(s), time=0.1) for s in (0.7, 0.3, 0.6)]
    return SimpleNamespace(dets=dets, out=out)


def test_pem_records_with_and_without_verification():
    from sam6d_b200 import pipeline
    f0, f1 = _frame(False), _frame(True)
    r0, r1 = pipeline.pem_records(f0), pipeline.pem_records(f1)
    base = (f0.out["pred_pose_score"] * f0.out["score"]).numpy()
    assert [r["score"] for r in r0] == [float(x) for x in base] and all("verify" not in r for r in r0)
    want = (f1.out["pred_pose_score"] * f1.out["score"] * f1.out["verify"]).numpy()
    assert [r["score"] for r in r1] == [float(x) for x in want]
    assert [r["verify"] for r in r1] == [float(x) for x in f1.out["verify"].numpy()]
    drop = lambda rs: [{k: v for k, v in r.items() if k not in ("score", "verify")} for r in rs]     # noqa: E731
    assert drop(r0) == drop(r1)
    assert np.array_equal(f1.pose_scores, want)
