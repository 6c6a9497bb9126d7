"""CPU: the COCO scoring definition of the BOP detection / segmentation tasks (oracle/bop_coco_oracle.py) on cases whose answers
are known by hand, the package's vectorised matching and accumulation (sam6d_b200/bop_eval_coco.py) against the oracle on seeded
random IoU matrices, the detection reader's errors and the CLI's argument errors."""
import json
import os

import numpy as np
import pytest

from oracle import bop_coco_oracle as bco
from sam6d_b200 import bop_eval_coco as bc
from sam6d_b200.cli import eval_bop_coco

import _bop_coco_split as split_mod

MED = 5000.0          # a medium area


def _oracle_one_category(images):
    """images: list of (ious, gt_ignore, gt_area, det_area, scores) of one category -> (precision, recall, stats)"""
    evals = [[]]
    evals[0] = [[] for _ in bco.AREA_RNGS]
    for ious, gi, ga, da, sc in images:
        for a, rng in enumerate(bco.AREA_RNGS):
            evals[0][a].append((list(sc), bco.evaluate_img(ious, gi, ga, da, rng)))
    p, r = bco.accumulate(evals, 1)
    return np.array(p), np.array(r), bco.summarize(p, r)


def test_perfect_detections():
    _, _, s = _oracle_one_category([([[1.0, 0.0], [0.0, 1.0]], [False, False], [MED, MED], [MED, MED], [0.9, 0.8])])
    assert s["AP"] == 1.0 and s["AR100"] == 1.0 and s["AP_medium"] == 1.0
    assert s["AP_small"] == -1.0 and s["AR_large"] == -1.0


def test_fp_tp_tp_gives_two_thirds():
    ious = [[0.0, 0.0], [1.0, 0.0], [0.0, 1.0]]           # FP, TP, TP in score order
    p, r, s = _oracle_one_category([(ious, [False, False], [MED, MED], [MED] * 3, [0.9, 0.8, 0.7])])
    assert (p[:, :, 0, 0, 2] == 2.0 / 3.0).all()           # rc = 0, 1/2, 1; pr = 0, 1/2, 2/3 -> 2/3 from the right
    assert s["AP"] == pytest.approx(2.0 / 3.0, abs=1e-15) and s["AR100"] == 1.0
    assert (r[:, 0, 0, 0] == 0.0).all()                    # maxDet 1 keeps the FP only
    # a detection on an ignored GT changes nothing
    ious2 = [[0.0, 0.0, 0.0], [0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]
    p2, r2, s2 = _oracle_one_category([(ious2, [False, False, True], [MED] * 3, [MED] * 4, [0.9, 0.85, 0.8, 0.7])])
    assert s2 == s and (p2[:, :, :, :, 2] == p[:, :, :, :, 2]).all()


def test_threshold_equality_and_ties():
    e = bco.evaluate_img([[0.5]], [False], [MED], [MED], bco.AREA_RNGS[0])
    assert e["gt_index"][0] == [0] and e["gt_index"][1] == [-1]     # IoU exactly 0.5 matches at t = 0.5, not at 0.55
    e = bco.evaluate_img([[0.7, 0.7]], [False, False], [MED, MED], [MED], bco.AREA_RNGS[0])
    assert e["gt_index"][0] == [1]                                    # an equal-IoU tie goes to the later GT
    # an ignored GT is scanned only when no non-ignored one matched
    e = bco.evaluate_img([[0.9, 0.6], [0.9, 0.0]], [True, False], [MED, MED], [MED, MED], bco.AREA_RNGS[0])
    assert [row for row in e["gt_index"][0]] == [1, 0] and e["det_ignore"][0] == [False, True]


def test_area_bounds_are_inclusive():
    for area, ranges in ((1024.0, (True, True, True, False)), (9216.0, (True, False, True, True)), (1023.0, (True, True, False, False))):
        for a, rng in enumerate(bco.AREA_RNGS):
            e = bco.evaluate_img([[1.0]], [False], [area], [area], rng)
            assert e["gt_ig"] == [not ranges[a]], (area, a)
    _, gi, ig = bc.match(np.ones((1, 1, 2)), [[False, False]], [[1024.0, 9216.0]], [[5000.0]])
    assert ig[0].tolist() == [[False, False], [False, True], [False, False], [True, False]]


def test_101st_detection_and_score_ties(tmp_path):
    split = split_mod.write_split(str(tmp_path), "toy", images=[(1, 0, 40, 50, [(1, 0.9, "")])])
    gt = split[(1, 0)][0][1]
    far = np.zeros_like(gt)
    far[0, 0] = True
    fps = [split_mod.record(1, 0, 1, 0.9, far) for _ in range(100)]
    path = lambda recs: split_mod.write_json(tmp_path / "r.json", recs)           # noqa: E731
    got = bco.evaluate(str(tmp_path), "toy", path(fps + [split_mod.record(1, 0, 1, 0.1, gt)]))
    assert got["AP"] == 0.0 and got["AR100"] == 0.0 and got["n_detections"] == 100         # the TP is the 101st: dropped
    got = bco.evaluate(str(tmp_path), "toy", path(fps[:99] + [split_mod.record(1, 0, 1, 0.1, gt)]))
    assert got["AR100"] == 1.0 and got["AP"] == pytest.approx(0.01, abs=1e-12)             # 1 / 100 at every threshold
    # equal scores keep file order: TP first -> AP 1 (1 / (1 + eps)); FP first -> precision 1/2
    tp, fp = split_mod.record(1, 0, 1, 0.5, gt), split_mod.record(1, 0, 1, 0.5, far)
    assert bco.evaluate(str(tmp_path), "toy", path([tp, fp]))["AP"] == pytest.approx(1.0, abs=1e-12)
    assert bco.evaluate(str(tmp_path), "toy", path([fp, tp]))["AP"] == pytest.approx(0.5, abs=1e-12)
    # bbox: the GT box is the full mask's, [x_min, y_min, w + 1, h + 1]
    b = split_mod.box_xywh(split[(1, 0)][0][2])
    got = bco.evaluate(str(tmp_path), "toy", path([split_mod.record(1, 0, 1, 0.5, gt, [float(v) for v in b])]), iou_type="bbox")
    assert got["AP"] == pytest.approx(1.0, abs=1e-12) and got["AR100"] == 1.0


def _random_case(rng, n_img, K):
    """random groups of K categories over n_img images; IoUs and areas from small grids so that ties, threshold-exact IoUs and
    area-range bounds occur"""
    grid = np.array([0.0, 0.3, 0.5, 0.55, 0.6, 0.7, 0.75, 0.8, 0.9, 0.95, 1.0])
    areas = np.array([10.0, 500.0, 1024.0, 3000.0, 9216.0, 20000.0])
    groups = []
    for i in range(n_img):
        for k in range(K):
            D, G = rng.randint(0, 12), rng.randint(0, 5)
            if D == 0 and G == 0:
                continue
            groups.append(dict(img=i, k=k, ious=grid[rng.randint(0, len(grid), (D, G))] * (rng.rand(D, G) < 0.6),
                               gi=rng.rand(G) < 0.25, ga=areas[rng.randint(0, len(areas), G)], da=areas[rng.randint(0, len(areas), D)],
                               sc=np.sort(np.round(rng.rand(D), 1))[::-1]))
    return groups


@pytest.mark.parametrize("seed", range(6))
def test_matching_and_accumulation_match_oracle(seed):
    rng = np.random.RandomState(seed)
    K = 3
    groups = _random_case(rng, 7, K)
    if seed % 2 == 0:
        for g in groups:                        # a category whose GT are all ignored: its cells hold -1
            if g["k"] == K - 1:
                g["gi"][:] = True
    # package: one batched match over the groups with both detections and GT
    A, T = len(bc.AREA_RNGS), len(bc.IOU_THRS)
    both = [g for g in groups if len(g["da"]) and len(g["ga"])]
    Dm = max(len(g["da"]) for g in both)
    Gm = max(len(g["ga"]) for g in both)
    I, gi, ga, da = np.zeros((len(both), Dm, Gm)), np.zeros((len(both), Gm), bool), np.zeros((len(both), Gm)), np.zeros((len(both), Dm))
    dv, gv = np.zeros((len(both), Dm), bool), np.zeros((len(both), Gm), bool)
    for j, g in enumerate(both):
        D, G = g["ious"].shape
        I[j, :D, :G], gi[j, :G], ga[j, :G], da[j, :D], dv[j, :D], gv[j, :G] = g["ious"], g["gi"], g["ga"], g["da"], True, True
    gidx, dig, _ = bc.match(I, gi, ga, da, dv, gv)
    evals = [[[] for _ in range(A)] for _ in range(K)]
    for j, g in enumerate(both):
        D = len(g["da"])
        for a, rngs in enumerate(bco.AREA_RNGS):
            e = bco.evaluate_img(g["ious"].tolist(), g["gi"].tolist(), g["ga"].tolist(), g["da"].tolist(), rngs)
            assert gidx[j, a, :, :D].tolist() == e["gt_index"], (seed, j, a)
            assert dig[j, a, :, :D].tolist() == e["det_ignore"], (seed, j, a)
    # accumulation: the groups image by image
    groups.sort(key=lambda g: (g["img"], g["k"]))
    pos = {id(g): j for j, g in enumerate(both)}
    sc, rk, ct, gc, gig = [], [], [], [], []
    dm, di = [], []
    lo, hi = bc.AREA_RNGS[:, 0], bc.AREA_RNGS[:, 1]
    for g in groups:
        D = len(g["da"])
        sc += g["sc"].tolist()
        rk += list(range(D))
        ct += [g["k"]] * D
        gc += [g["k"]] * len(g["ga"])
        gig.append(g["gi"][None, :] | (g["ga"][None, :] < lo[:, None]) | (g["ga"][None, :] > hi[:, None]))
        if id(g) in pos:
            j = pos[id(g)]
            dm.append(gidx[j, :, :, :D] >= 0)
            di.append(dig[j, :, :, :D])
        else:
            dm.append(np.zeros((A, T, D), bool))
            di.append(np.broadcast_to(((g["da"][None, :] < lo[:, None]) | (g["da"][None, :] > hi[:, None]))[:, None, :], (A, T, D)))
        for a, rngs in enumerate(bco.AREA_RNGS):
            evals[g["k"]][a].append((g["sc"].tolist(), bco.evaluate_img(g["ious"].tolist(), g["gi"].tolist(), g["ga"].tolist(),
                                                                        g["da"].tolist(), rngs)))
    p, r = bc.accumulate(np.array(sc), np.array(rk), np.array(ct), np.concatenate(dm, 2), np.concatenate(di, 2), np.array(gc),
                         np.concatenate(gig, 1), K)
    po, ro = bco.accumulate(evals, K)
    np.testing.assert_array_equal(p, np.array(po))
    np.testing.assert_array_equal(r, np.array(ro))
    assert ((p > 0) & (p < 1)).any() and (p == 0).any()
    assert ((p[:, :, K - 1] == -1).all() and (r[:, K - 1] == -1).all()) == (seed % 2 == 0)
    s, so = bc.summarize(p, r), bco.summarize(po, ro)
    assert list(s) == list(bc.STAT_NAMES) == bco.STAT_NAMES
    for k in s:
        assert abs(s[k] - so[k]) <= 1e-12, (k, s[k], so[k])


def test_bbox_iou_matches_oracle():
    rng = np.random.RandomState(3)
    d = np.round(rng.uniform(0, 40, (30, 4)), 1)
    g = np.round(rng.uniform(0, 40, (7, 4)), 0)
    g[0] = [5, 5, 0, 10]                                   # zero width
    got = bc.bbox_iou(d, g)
    want = [[bco.bbox_iou(a.tolist(), b.tolist()) for b in g] for a in d]
    np.testing.assert_array_equal(got, want)
    assert (got > 0).any()


def test_run_lists():
    m = np.zeros((3, 4), np.uint8)
    m[0, 0], m[2, 0], m[0, 1], m[1, 3], m[2, 3] = 1, 7, 255, 2, 3
    runs, box = bco.mask_runs(m)
    assert runs == [(0, 1), (2, 4), (10, 12)] and box == (0, 0, 3, 2)
    rle = split_mod.mask_to_rle(m > 0)
    assert bco.rle_runs(rle["counts"]) == runs and bc.rle_area(rle["counts"]) == 5
    assert bco.runs_intersection(runs, [(1, 3), (11, 20)]) == 2


def test_reader_errors(tmp_path):
    good = split_mod.record(1, 0, 1, 0.5, np.eye(4, 5, dtype=bool))
    p = tmp_path / "r.json"
    p.write_text(json.dumps([good]))
    d = bc.load_detections(str(p))
    assert d["obj_id"].tolist() == [1] and d["size"].tolist() == [[4, 5]] and bc.rle_area(d["counts"][0]) == 4
    cases = [({"scene_id": "1"}, "record 1: scene_id"), ({"image_id": None}, "record 1: image_id"), ({"category_id": 1.5}, "category_id"),
             ({"score": float("nan")}, "record 1: score"), ({"bbox": [1, 2, 3]}, "record 1: bbox"),
             ({"segmentation": {"counts": [1, 2]}}, "record 1: segmentation"),
             ({"segmentation": {"counts": [3, 2], "size": [4, 5]}}, "record 1: segmentation counts"),
             ({"segmentation": {"counts": [25, -5, 0], "size": [4, 5]}}, "non-negative"),
             ({"segmentation": {"counts": [20], "size": [4, 0]}}, "size")]
    for change, msg in cases:
        p.write_text(json.dumps([good, dict(good, **change)]))
        with pytest.raises(ValueError, match=msg):
            bc.load_detections(str(p))
    p.write_text(json.dumps([dict(good, segmentation={"counts": "abc", "size": [4, 5]})]))
    with pytest.raises(NotImplementedError, match="record 0"):
        bc.load_detections(str(p))
    p.write_text(json.dumps({"a": 1}))
    with pytest.raises(ValueError, match="list"):
        bc.load_detections(str(p))
    with pytest.raises(ValueError, match="iou_type"):
        bc.evaluate_bop22_coco(str(tmp_path), "toy", str(p), iou_type="keypoints")
    with pytest.raises(ValueError, match="bbox_type"):
        bc.evaluate_bop22_coco(str(tmp_path), "toy", str(p), bbox_type="tight")


def test_cli_argument_errors(tmp_path, capsys):
    res = tmp_path / "r.json"
    base = ["--bop_root", str(tmp_path), "--output_dir", str(tmp_path / "out")]
    ds = tmp_path / "toy"
    ds.mkdir()

    def fails(args, msg):
        with pytest.raises(SystemExit) as e:
            eval_bop_coco.main(base + args)
        assert e.value.code == 2 and msg in capsys.readouterr().err
    fails(["--dataset_name", "missing", "--result_json", str(res)], "no dataset directory")
    fails(["--dataset_name", "toy", "--result_json", str(res)], "no test split directory")
    (ds / "test").mkdir()
    fails(["--dataset_name", "toy", "--result_json", str(res), "--targets", str(tmp_path / "none.json")], "no targets file")
    (ds / "test_targets_bop19.json").write_text("[]")
    fails(["--dataset_name", "toy", "--result_json", str(res)], "no results file")
    fails(["--dataset_name", "toy", "--result_json", str(res), "--iou_type", "keypoints"], "--iou_type")
    fails(["--dataset_name", "toy", "--result_json", str(res), "--bbox_type", "tight"], "--bbox_type")
