"""CPU: the BOP19 scoring definitions (oracle/bop_eval_oracle.py) on cases whose answers are known by hand, the host halves of
sam6d_b200/bop_eval.py against them (symmetry sets, sphere test, VSD errors from counts, matching), the readers and the CLI's
argument errors."""
import json
import math
import os

import numpy as np
import pytest

from oracle import bop_eval_oracle as bo
from sam6d_b200 import bop_eval as be
from sam6d_b200.cli import eval_bop

FLIP_X = [1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1]      # 180 degrees about x
FLIP_Z = [-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]      # 180 degrees about z
CONT_Z = {"axis": [0, 0, 1], "offset": [0, 0, 0]}


def _box(a=10.0, b=20.0, c=30.0):
    return np.array([[x, y, z] for x in (-a, a) for y in (-b, b) for z in (-c, c)], np.float64)


@pytest.mark.parametrize("info,n", [({}, 1), ({"symmetries_discrete": [FLIP_X]}, 2), ({"symmetries_discrete": [FLIP_X, FLIP_Z]}, 3),
                                    ({"symmetries_continuous": [CONT_Z]}, 314),
                                    ({"symmetries_continuous": [CONT_Z], "symmetries_discrete": [FLIP_X]}, 628),
                                    ({"symmetries_continuous": [CONT_Z], "symmetries_discrete": [FLIP_X, FLIP_Z]}, 942)])
def test_symmetry_set_sizes(info, n):
    syms = bo.symmetries(info)
    R, t = be.symmetry_transforms(info)
    assert len(syms) == n and R.shape == (n, 3, 3) and t.shape == (n, 3)
    np.testing.assert_allclose(R, np.stack([s[0] for s in syms]), atol=1e-14)
    np.testing.assert_allclose(t, np.stack([s[1] for s in syms]), atol=1e-12)
    for Ri in R:
        np.testing.assert_allclose(Ri @ Ri.T, np.eye(3), atol=1e-12)
    has_identity = any(np.array_equal(Ri, np.eye(3)) and not t[i].any() for i, Ri in enumerate(R))
    assert has_identity == ("symmetries_continuous" not in info)
    if "symmetries_continuous" in info:
        # not even approximately: with the continuous set alone the nearest element is one step of 2 pi / 315 away; a flip
        # about the same axis adds the rotations by pi + i 2 pi / 315, half a step off the grid (315 is odd)
        ang = min(math.acos(max(-1.0, min(1.0, (np.trace(Ri) - 1) / 2))) for Ri in R)
        step = 2 * math.pi / 315
        assert ang == pytest.approx(step / 2 if FLIP_Z in info.get("symmetries_discrete", []) else step, rel=1e-9)


def test_continuous_offset_fixes_the_axis():
    info = {"symmetries_continuous": [{"axis": [0, 1, 0], "offset": [5.0, 0.0, -3.0]}]}
    for Rs, ts in bo.symmetries(info):
        np.testing.assert_allclose(Rs @ np.array([5.0, 7.0, -3.0]) + ts, [5.0, 7.0, -3.0], atol=1e-12)


def test_pure_translation():
    X = _box()
    R = np.eye(3)
    t_g = np.array([0.0, 0.0, 500.0])
    d = np.array([3.0, -4.0, 0.0])
    syms = bo.symmetries({})
    assert bo.mssd(R, t_g + d, R, t_g, X, syms) == pytest.approx(5.0, abs=1e-12)
    # every vertex moves by (3, -4) mm at its own depth z: |du, dv| = f 5 / z, largest at the nearest z = 470
    K = [[600.0, 0, 320], [0, 600.0, 240], [0, 0, 1]]
    assert bo.mspd(R, t_g + d, R, t_g, X, syms, K) == pytest.approx(600.0 * 5.0 / 470.0, rel=1e-12)
    # a shift along the optical axis moves a vertex's projection by f |x| (1/z - 1/(z + dz))
    d = np.array([0.0, 0.0, 30.0])
    want = max(math.hypot(600 * x * (1 / (500 + z) - 1 / (530 + z)), 600 * y * (1 / (500 + z) - 1 / (530 + z))) for x, y, z in X)
    assert bo.mspd(R, t_g + d, R, t_g, X, syms, K) == pytest.approx(want, rel=1e-12)


def _rz(a):
    return bo.rotation([0, 0, 1], a)


def test_mssd_symmetry_steps():
    X = _box(15.0, 15.0, 40.0)
    info = {"symmetries_continuous": [CONT_Z]}
    syms = bo.symmetries(info)
    R_g, t_g = bo.rotation([1, 2, 3], 0.7), np.array([10.0, -20.0, 600.0])
    step = 2 * math.pi / 315
    # on the grid: R_e = R_g R_s
    assert bo.mssd(R_g @ _rz(7 * step), t_g, R_g, t_g, X, syms) < 1e-9
    # off the grid (not next to the missing identity): at most the chord of half a step at the largest radius from the axis
    r = float(np.hypot(X[:, 0], X[:, 1]).max())
    bound = 2 * r * math.sin(step / 4)
    for frac in (0.5, 0.3, 0.81):
        e = bo.mssd(R_g @ _rz((7 + frac) * step), t_g, R_g, t_g, X, syms)
        assert 0 < e <= bound * (1 + 1e-9)
    assert bo.mssd(R_g @ _rz(7.5 * step), t_g, R_g, t_g, X, syms) == pytest.approx(bound, rel=1e-9)
    # est = GT: the set has no identity, so the error is one whole step's chord
    assert bo.mssd(R_g, t_g, R_g, t_g, X, syms) == pytest.approx(2 * r * math.sin(step / 2), rel=1e-9)


def test_vsd_hand_made_counts():
    K = np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1]])       # pixel (u, v) at factor sqrt(u^2 + v^2 + 1)
    f = np.sqrt(np.arange(3)[None, :] ** 2 + np.arange(2)[:, None] ** 2 + 1.0)
    dist_g = np.array([[100, 100, 0], [100, 100, 100]], np.float64)
    dist_e = np.array([[100, 104, 100], [0, 100, 128]], np.float64)
    dist_t = np.array([[100, 100, 0], [100, 50, 100]], np.float64)
    # V_g: d_g > 0 and (d_g - d_t <= 15 or d_t = 0): (1,1) is occluded (100 - 50 > 15)
    # V_e: (0,2) has d_t = 0 -> visible; (1,1) 100 - 50 > 15 and not in V_g -> not; (1,2) 128 - 100 > 15 but V_g and d_e > 0 -> visible
    # U = {(0,0),(0,1),(0,2),(1,0),(1,2)} = 5, I = {(0,0),(0,1),(1,2)} = 3; |d_g - d_e| / 100 on I: 0, 0.04, 0.28
    c = bo.vsd_counts(dist_e / f, dist_g / f, dist_t / f, K, 15.0, 100.0)
    assert c[:2] == [5, 3]
    assert c[2:] == [1, 1, 1, 1, 1, 0, 0, 0, 0, 0]          # 0.28 >= tau for tau <= 0.25
    e = bo.vsd_errors(c)
    assert e[0] == pytest.approx((1 + 2) / 5) and e[-1] == pytest.approx(2 / 5)
    np.testing.assert_allclose(be.vsd_errors(np.array([c])), [e])
    assert be.vsd_errors(np.zeros((1, 12))).tolist() == [[1.0] * 10]


def test_vsd_identical_unoccluded_is_zero():
    K = np.array([[500.0, 0, 8], [0, 500.0, 6], [0, 0, 1]])
    d = np.zeros((12, 16))
    d[3:9, 4:12] = 700.0 + np.arange(8)[None, :]
    c = bo.vsd_counts(d, d, d, K, 15.0, 80.0)
    assert c[0] == c[1] == 48 and c[2:] == [0] * 10
    assert bo.vsd_errors(c) == [0.0] * 10


def test_sphere_test():
    r = 50.0
    assert bo.spheres_overlap([0, 0, 1000], [0, 0, 1000], r)
    assert not bo.spheres_overlap([0, 0, 1000], [101, 0, 1000], r)        # 0.101 > 0.05 + 0.05
    assert bo.spheres_overlap([0, 0, 1000], [99, 0, 1000], r)
    te = np.array([[0, 0, 1000], [0, 0, 1000], [0, 0, 1000]], np.float64)
    tg = np.array([[0, 0, 1000], [101, 0, 1000], [99, 0, 1000]], np.float64)
    assert be.spheres_overlap(te, tg, np.full(3, r)).tolist() == [True, False, True]


def _match_both(err, valid, thr):
    a = bo.match(err, valid, thr)
    b = be.match_count(np.asarray(err, np.float64)[None], np.array([thr]), np.asarray(valid))[0]
    assert a == b
    return a


def test_matching_cases():
    # two instances; the higher-scored estimate is closer to GT 1 but also below the threshold for GT 0
    err = [[3.0, 1.0],      # estimate 0 (highest score) takes GT 1, its smallest error
           [2.0, 0.5]]      # estimate 1 is left with GT 0
    assert _match_both(err, [True, True], 4.0) == 2
    assert _match_both(err, [True, True], 2.5) == 2
    assert _match_both(err, [True, True], 1.5) == 1      # estimate 1's only candidate below 1.5 (GT 1) is taken
    # score order beats error order: estimate 0 claims GT 0 although estimate 1 fits it better
    assert _match_both([[1.0, 9.0], [0.1, 9.0]], [True, True], 2.0) == 1
    # an invalid GT (visib_fract < 0.1) takes a match and counts nothing
    assert _match_both([[0.5, 1.0], [0.6, 9.0]], [False, True], 2.0) == 0     # estimate 1 has nothing left below 2
    assert _match_both([[0.5, 1.0], [0.6, 1.5]], [False, True], 2.0) == 1
    assert _match_both([[0.5], [0.6]], [False], 2.0) == 0
    # the threshold is strict
    assert _match_both([[2.0]], [True], 2.0) == 0
    # ties go to the first GT
    a = be.match_count(np.array([[[1.0, 1.0]]]), np.array([2.0]), np.array([False, True]))
    assert a.tolist() == [0]


def _write_split(root, n_extra_results=0):
    ds = os.path.join(root, "toy")
    os.makedirs(os.path.join(ds, "models_eval"))
    with open(os.path.join(ds, "models_eval", "models_info.json"), "w") as fh:
        json.dump({"1": {"diameter": 100.0}, "2": {"diameter": 50.0, "symmetries_continuous": [CONT_Z]}}, fh)
    with open(os.path.join(ds, "test_targets_bop19.json"), "w") as fh:
        json.dump([{"scene_id": 1, "im_id": 3, "obj_id": 1, "inst_count": 2}], fh)
    return ds


def test_readers(tmp_path):
    ds = _write_split(str(tmp_path))
    assert be.load_targets(os.path.join(ds, "test_targets_bop19.json")) == [(1, 3, 1, 2)]
    info = be.load_models_info(os.path.join(ds, "models_eval", "models_info.json"))
    assert info[1]["diameter"] == 100.0 and len(be.symmetry_transforms(info[2])[0]) == 314
    csv = tmp_path / "r.csv"
    rows = ["scene_id,im_id,obj_id,score,R,t,time\n", "1,3,1,0.5,1 0 0 0 1 0 0 0 1,1.5 -2 700,0.25\n",
            "1,3,2,0.75,0 -1 0 1 0 0 0 0 1,0 0 650.5,0.25\n"]
    csv.write_text("".join(rows))
    r = be.load_results(str(csv))
    assert r["scene_id"].tolist() == [1, 1] and r["obj_id"].tolist() == [1, 2] and r["score"].tolist() == [0.5, 0.75]
    np.testing.assert_array_equal(r["R"][1], [[0, -1, 0], [1, 0, 0], [0, 0, 1]])
    np.testing.assert_array_equal(r["t"][0], [1.5, -2, 700])
    csv.write_text("".join(rows[1:]))                     # no header: bop.csv_rows writes none
    assert len(be.load_results(str(csv))["score"]) == 2
    csv.write_text("1,3,1,0.5,1 0 0 0 1 0 0 0,1 2 3,0\n")
    with pytest.raises(ValueError, match=":1:"):
        be.load_results(str(csv))
    bad = tmp_path / "t.json"
    bad.write_text(json.dumps([{"scene_id": 1, "im_id": 2}]))
    with pytest.raises(ValueError, match="inst_count"):
        be.load_targets(str(bad))


def test_models_dir_fallback_warns(tmp_path):
    ds = tmp_path / "tless"
    (ds / "models_cad").mkdir(parents=True)
    with pytest.warns(UserWarning, match="models_cad"):
        assert be.models_eval_dir(str(tmp_path), "tless") == str(ds / "models_cad")
    (ds / "models_eval").mkdir()
    assert be.models_eval_dir(str(tmp_path), "tless") == str(ds / "models_eval")


def test_cli_argument_errors(tmp_path, capsys):
    ds = _write_split(str(tmp_path))
    csv = tmp_path / "r.csv"
    base = ["--bop_root", str(tmp_path), "--output_dir", str(tmp_path / "out")]
    with pytest.raises(SystemExit) as e:
        eval_bop.main(base + ["--dataset_name", "missing", "--result_csv", str(csv)])
    assert e.value.code == 2 and "no dataset directory" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        eval_bop.main(base + ["--dataset_name", "toy", "--result_csv", str(csv)])
    assert e.value.code == 2 and "no test split directory" in capsys.readouterr().err
    os.makedirs(os.path.join(ds, "test"))
    with pytest.raises(SystemExit) as e:
        eval_bop.main(base + ["--dataset_name", "toy", "--result_csv", str(csv), "--targets", str(tmp_path / "none.json")])
    assert e.value.code == 2 and "no targets file" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        eval_bop.main(base + ["--dataset_name", "toy", "--result_csv", str(csv)])
    assert e.value.code == 2 and "no results file" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        eval_bop.main(base + ["--dataset_name", "toy", "--result_csv", str(csv), "--error_types", "add"])
    assert e.value.code == 2
