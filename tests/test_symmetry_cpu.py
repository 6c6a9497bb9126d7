"""CPU: the symmetry finder (sam6d_b200/symmetry.py) on the float64 oracle backend (oracle/symmetry_oracle.py), its models_info
output, the symmetric pick's oracle, and the argument checks of find_symmetries, onboard_objects and the two CLIs."""
import math
import os
import sys

import numpy as np
import pytest

from oracle import hypotheses_oracle as ho
from oracle import symmetry_oracle as so

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _symmetry_meshes as sm                                                  # noqa: E402

from sam6d_b200 import bop_eval, symmetry                                      # noqa: E402


def _check(info, name, rot):
    nd, axis = sm.EXPECTED[name]
    assert len(info.get("symmetries_discrete", [])) == nd, (name, len(info.get("symmetries_discrete", [])))
    cont = info.get("symmetries_continuous", [])
    if axis is None:
        assert not cont, name
        return
    assert len(cont) == 1
    assert abs(abs(float(np.dot(cont[0]["axis"], rot @ np.asarray(axis)))) - 1.0) < 1e-3


@pytest.mark.parametrize("placement", ["as_built", "moved"])
@pytest.mark.parametrize("name", sm.NAMES)
def test_expected_groups_on_the_oracle(name, placement):
    rot = np.eye(3) if placement == "as_built" else sm.random_rotation()
    mesh = sm.build(name) if placement == "as_built" else sm.placed(sm.build(name), rot)
    info, det = symmetry.find_symmetries(mesh, backend=so.Float64Backend(), return_details=True)
    _check(info, name, rot)
    # every reported transform maps the surface onto itself: its agreement passes, and t = c - R c
    c = det["centre"]
    for m in info.get("symmetries_discrete", []):
        m = np.asarray(m).reshape(4, 4)
        assert np.allclose(m[:3, :3] @ m[:3, :3].T, np.eye(3), atol=1e-9) and np.isclose(np.linalg.det(m[:3, :3]), 1.0)
        assert np.allclose(m[:3, 3], c - m[:3, :3] @ c, atol=1e-6)
        assert np.allclose(m[3], [0, 0, 0, 1])
    # the models_info output round-trips through bop_eval.symmetry_transforms
    R, t = bop_eval.symmetry_transforms(info)
    nd, axis = sm.EXPECTED[name]
    assert R.shape == ((1 + nd) * (1 if axis is None else 314), 3, 3)
    assert np.allclose(np.einsum("sij,skj->sik", R, R), np.eye(3), atol=1e-9)
    print(f"{name} {placement}: identity count {det['identity_count']}, threshold {det['threshold']:.0f}, orders {det['orders']}")


def test_margins_of_the_defaults():
    """the passing elements of the cube sit well above the threshold and the failing rotations well below it"""
    mesh = sm.build("cube")
    info, det = symmetry.find_symmetries(mesh, backend=so.Float64Backend(), return_details=True)
    counts = det["stage1_counts"][1:]
    thr = det["threshold"]
    passing, failing = counts[counts >= thr], counts[counts < thr]
    print(f"cube stage 1: identity {det['identity_count']}, threshold {thr:.0f}, weakest pass {passing.min()}, strongest fail {failing.max()}")
    assert passing.min() - thr > 0.03 * symmetry.N_QUERY and thr - failing.max() > 0.3 * symmetry.N_QUERY


def test_models_info_entry_and_pick_set():
    mesh = sm.placed(sm.build("cylinder"), sm.random_rotation(5))
    info = symmetry.models_info_entry(mesh, backend=so.Float64Backend())
    v = np.asarray(mesh.vertices, np.float64)
    assert np.isclose(info["diameter"], so.diameter(v.astype(np.float32)))
    for k, ax in enumerate("xyz"):
        assert np.isclose(info[f"min_{ax}"], v[:, k].min()) and np.isclose(info[f"size_{ax}"], np.ptp(v[:, k]))
    R, t = symmetry.pick_set(info)
    # identity first, the discrete flip, then 71 steps of 5 degrees composed with identity and flip
    assert len(R) == 2 + 2 * 71 and np.array_equal(R[0], np.eye(3)) and np.array_equal(t[0], np.zeros(3))
    m = np.asarray(info["symmetries_discrete"][0]).reshape(4, 4)
    assert np.allclose(R[1], m[:3, :3]) and np.allclose(t[1], m[:3, 3] / 1000.0)
    axis = np.asarray(info["symmetries_continuous"][0]["axis"])
    ang = [math.degrees(math.acos(np.clip((np.trace(r) - 1) / 2, -1, 1))) for r in R[2:2 + 71]]
    assert np.allclose(sorted(min(a, 360 - a) for a in ang)[:2], [5.0, 5.0], atol=1e-6)
    assert all(np.allclose(r @ axis, axis) for r in R[2:2 + 71])
    assert symmetry.pick_set({})[0].shape == (1, 3, 3)


def test_group_closure_matches_the_oracle():
    from sam6d_b200.bop_eval import _axis_angle
    gens = [_axis_angle(np.array([0, 0, 1.0]), math.pi / 2), _axis_angle(np.array([1.0, 0, 0]), math.pi / 2)]
    a, b = symmetry.close_group(gens), so.close_group(gens)
    assert len(a) == len(b) == 24
    assert all(any(np.allclose(x, y, atol=1e-9) for y in b) for x in a)
    hexa = [_axis_angle(np.array([0, 0, 1.0]), math.pi / 3), _axis_angle(np.array([1.0, 0, 0]), math.pi)]
    assert len(symmetry.close_group(hexa)) == len(so.close_group(hexa)) == 12


def test_sym_pick_oracle_with_identity_ranges_is_the_plain_pick():
    rng = np.random.default_rng(0)
    from scipy.spatial.transform import Rotation
    B, n2, K = 3, 40, 6
    Rt = np.concatenate([Rotation.random(B * n2, random_state=1).as_matrix().reshape(B, n2, 9),
                         rng.normal(0, 0.3, (B, n2, 3))], axis=2).astype(np.float32)
    top = np.tile(np.arange(n2, dtype=np.int32), (B, 1))
    scores = rng.random((B, n2)).astype(np.float32)
    ct, dm = ho.thresholds(60.0, 0.3)
    R, t, valid, count = so.pick_distinct_sym(Rt, top, scores, K, ct, dm, np.eye(3).reshape(1, 9), np.zeros((1, 3)),
                                              np.zeros((B, 2), np.int32) + [0, 1], np.full(B, 0.07, np.float32))
    R2, t2, _, valid2, count2, _, _ = ho.pick_distinct(Rt, top, scores, K, ct, dm, fp32=True)
    assert np.array_equal(count, count2) and np.array_equal(valid, valid2) and np.array_equal(R, R2.astype(np.float32))


# ---- argument checks ---------------------------------------------------------------------------------------------------------
def test_find_symmetries_argument_checks():
    mesh = sm.build("cube")
    for kw in (dict(geo_tol=0.0), dict(geo_tol=float("nan")), dict(color_tol=-0.1), dict(slack=2.0), dict(geo_tol=True),
               dict(slack="0.1")):
        with pytest.raises(ValueError):
            symmetry.find_symmetries(mesh, backend=so.Float64Backend(), **kw)
    flat = sm._mesh(np.zeros((3, 3)), np.zeros((0, 3)))
    with pytest.raises(ValueError, match="faces"):
        symmetry.find_symmetries(flat, backend=so.Float64Backend())
    with pytest.raises(ValueError, match="area"):
        symmetry.find_symmetries(sm._mesh(np.zeros((3, 3)), [[0, 1, 2]]), backend=so.Float64Backend())


def test_pack_sets_cap():
    big = {"symmetries_discrete": [list(np.eye(4).reshape(-1))] * 2048}
    with pytest.raises(ValueError, match="at most"):
        symmetry.pack_sets([big], "cpu")
    s = symmetry.pack_sets([{}, {"symmetries_discrete": [list(np.eye(4).reshape(-1))]}], "cpu")
    assert s.range.tolist() == [[0, 1], [1, 2]] and tuple(s.R.shape) == (3, 3, 3)


def test_onboard_objects_argument_checks():
    from sam6d_b200 import pipeline
    model = pipeline.SAM6D.__new__(pipeline.SAM6D)
    model.rendering_type = "pyrender"
    for bad in ("models_info", "yes", 3, {1: {}}, {1: {}, 2: "x"}):
        with pytest.raises(ValueError, match="symmetries"):
            model.onboard_objects([sm.build("cube"), sm.build("cone")], obj_ids=[1, 2], symmetries=bad)
    pipeline.check_symmetries({1: {}, 2: {}}, [1, 2])
    pipeline.check_symmetries("models_info", [1], pipeline.SYMMETRY_SOURCES + ("models_info",))


def test_cli_argument_checks(tmp_path, capsys):
    from sam6d_b200.cli import make_models_info, pem_run_inference_custom, run_bop, run_sam6d
    ply = tmp_path / "a.ply"
    ply.write_text("ply\n")
    out = str(tmp_path / "mi.json")
    for args in ([], ["--cad_path", str(ply), "--models_dir", str(tmp_path)], ["--cad_path", str(ply), "--obj_ids", "1", "2"],
                 ["--cad_path", str(ply), str(ply), "--obj_ids", "3", "3"], ["--models_dir", str(tmp_path / "none")],
                 ["--models_dir", str(tmp_path), "--obj_ids", "1"], ["--cad_path", str(tmp_path / "missing.ply")],
                 ["--cad_path", str(ply), "--geo_tol", "0"], ["--cad_path", str(ply), "--slack", "nan"]):
        with pytest.raises(SystemExit):
            make_models_info.main(args + ["--output", out])
    assert not os.path.exists(out)
    common = ["--output_dir", str(tmp_path), "--cad_path", str(ply), "--rgb_path", "x", "--depth_path", "x", "--cam_path", "x"]
    for cli, extra in ((run_sam6d, []), (pem_run_inference_custom, ["--seg_path", "x"])):
        with pytest.raises(SystemExit):
            cli.main(common + extra + ["--pem_hypotheses", "4", "--hyp_symmetries", "models_info"])
        assert "models_info" in capsys.readouterr().err
        with pytest.raises(SystemExit):
            cli.main(common + extra + ["--hyp_symmetries", "sometimes"])
    # run_bop takes models_info: the run stops at the missing dataset, not at the option
    with pytest.raises(SystemExit):
        run_bop.main(["--bop_root", str(tmp_path), "--dataset_name", "nope", "--output_dir", str(tmp_path), "--stage", "pem",
                      "--template_dir", str(tmp_path), "--pem_hypotheses", "4", "--hyp_symmetries", "models_info"])
    err = capsys.readouterr().err
    assert "no dataset directory" in err and "only run_bop" not in err
