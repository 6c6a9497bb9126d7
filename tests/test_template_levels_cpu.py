"""CPU: the ISM's template view sets (render.template_poses / template_view_set) against the reference's CNOS level-0 / 1 / 2
poses (tests/golden/template_poses_level0.pt, template_poses_levels.pt: tools/make_golden_render.py,
tools/make_golden_template_levels.py), and the view-set / aggregation options of the CLIs and SAM6D."""
import os

import numpy as np
import pytest
import torch

from sam6d_b200 import render


def _reference(golden_dir, level):
    if level == 0:
        g = torch.load(os.path.join(golden_dir, "template_poses_level0.pt"))
        return g["cam_poses"].numpy(), g["obj_poses"].numpy()
    g = torch.load(os.path.join(golden_dir, "template_poses_levels.pt"))
    return g[f"cam_poses_level{level}"].numpy(), g[f"obj_poses_level{level}"].numpy()


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("dist", ["all", "upper"])
def test_template_poses_match_reference_as_a_set(golden_dir, level, dist):
    cam, obj = _reference(golden_dir, level)
    ref = obj if dist == "all" else obj[cam[:, 2, 3] >= 0]                 # get_obj_poses_from_template_level's "upper" rule
    ours = render.template_poses(level, dist, 1000.0)
    assert len(ours) == {0: 42, 1: 162, 2: 642}[level] if dist == "all" else len(ours) == {0: 26, 1: 91, 2: 341}[level]
    assert len(ours) == len(ref)
    d = np.abs(ours[:, None, :3, :3] - ref[None, :, :3, :3]).max(axis=(2, 3))
    match = d.argmin(axis=1)
    assert sorted(match.tolist()) == list(range(len(ref)))                           # a bijection
    assert d.min(axis=1).max() < 1e-5
    assert np.abs(ours[:, :3, 3] - ref[match, :3, 3]).max() < 1e-3                  # (0, 0, 1000) up to rounding
    R = ours[:, :3, :3]
    assert np.allclose(R @ R.transpose(0, 2, 1), np.eye(3), atol=1e-12) and np.allclose(np.linalg.det(R), 1.0, atol=1e-12)
    # camera directions of the reference's Blender icosphere
    c = render.camera_centres(ours) / 1000.0
    rc = cam[:, :3, 3] / np.linalg.norm(cam[:, :3, 3], axis=1, keepdims=True)
    rc = rc if dist == "all" else rc[cam[:, 2, 3] >= 0]
    assert np.linalg.norm(c[:, None] - rc[None], axis=2).min(axis=1).max() < 2e-5


@pytest.mark.parametrize("level", [0, 1, 2])
def test_order_is_elevation_then_azimuth_and_upper_is_z_nonnegative(level):
    for dist in ("all", "upper"):
        P = render.template_poses(level, dist, 2.0)
        cam = render.camera_centres(P)
        np.testing.assert_allclose(np.linalg.norm(cam, axis=1), 2.0, atol=1e-12)
        el = np.round(np.degrees(np.arctan2(cam[:, 2], np.hypot(cam[:, 0], cam[:, 1]))), 6)
        az = np.round(np.degrees(np.arctan2(cam[:, 0], cam[:, 1])), 6)
        keys = list(zip(el, az))
        assert keys == sorted(keys)
        if dist == "upper":
            assert (el >= 0).all() and (el == 0).sum() == 10 * 2 ** level          # the equator ring is kept
            np.testing.assert_array_equal(P, [p for p in render.template_poses(level, "all", 2.0) if render.camera_centres(p[None])[0, 2] >= -1e-9])


def test_level0_is_level0_template_poses():
    for d in (1.0, 400.0):
        np.testing.assert_array_equal(render.template_poses(0, "all", d), render.level0_template_poses(d))


@pytest.mark.parametrize("level", [0, 1, 2])
def test_reference_level_indices_in_level2_name_the_same_views(golden_dir, level):
    """load_index_level_in_level2(level, "all") picks, among the level-2 poses, the level's own views: ours at level 2 indexed
    the same way are ours at that level"""
    g = torch.load(os.path.join(golden_dir, "template_poses_levels.pt"))
    if level == 2:
        return
    idx = g[f"idx_all_level{level}_in_level2"].numpy()
    ref2 = g["obj_poses_level2"].numpy()[idx]
    ours = render.template_poses(level, "all", 1000.0)
    d = np.abs(ours[:, None, :3, :3] - ref2[None, :, :3, :3]).max(axis=(2, 3))
    assert sorted(d.argmin(axis=1).tolist()) == list(range(len(idx))) and d.min(axis=1).max() < 1e-5


@pytest.mark.parametrize("level,dist,n_union,n_ism", [(0, "all", 42, 42), (0, "upper", 42, 26), (1, "all", 162, 162),
                                                       (1, "upper", 107, 91), (2, "all", 642, 642), (2, "upper", 357, 341)])
def test_view_set_puts_level0_first(level, dist, n_union, n_ism):
    union, idx = render.template_view_set(level, dist, 3.0)
    assert union.shape == (n_union, 4, 4) and idx.shape == (n_ism,) and idx.dtype == np.int64
    np.testing.assert_array_equal(union[:42], render.level0_template_poses(3.0))          # rgb_0..41 are today's views
    np.testing.assert_array_equal(union[idx], render.template_poses(level, dist, 3.0))   # the ISM's views, in the set's order
    assert len(set(idx.tolist())) == n_ism
    assert set(range(42, n_union)) <= set(idx.tolist())                                    # nothing rendered for nobody
    cam = render.camera_centres(union)
    assert np.linalg.norm(cam[:, None] - cam[None], axis=2)[~np.eye(n_union, dtype=bool)].min() > 1e-3   # no view twice
    if (level, dist) == (0, "all"):
        np.testing.assert_array_equal(idx, np.arange(42))


def test_view_set_rejects_unknown_settings():
    for bad in ((3, "all"), (-1, "all"), (0, "lower")):
        with pytest.raises(ValueError):
            render.template_view_set(*bad)


def test_render_cli_view_set_flags(tmp_path, golden_dir):
    from sam6d_b200.cli import render_bop_templates as bop, render_custom_templates as cli
    a = cli.parse_args(["--cad_path", "x.ply", "--output_dir", "o"])
    assert (a.level_templates, a.pose_distribution, a.size, a.poses) == (0, "all", 512, None)
    a = cli.parse_args(["--cad_path", "x.ply", "--output_dir", "o", "--level_templates", "2", "--pose_distribution", "upper"])
    assert (a.level_templates, a.pose_distribution, a.cad_path) == (2, "upper", "x.ply")
    a = bop.parse_args(["--dataset_name", "ycbv", "--level_templates", "1"])
    assert (a.dataset_name, a.level_templates, a.pose_distribution) == ("ycbv", 1, "all")
    for bad in (["--level_templates", "3"], ["--pose_distribution", "lower"], ["--no_such_flag"]):
        with pytest.raises(SystemExit):
            cli.parse_args(["--cad_path", "x.ply"] + bad)
    # the defaults render today's 42 views; a poses file keeps its own views and takes no view-set flags
    P, idx = cli.view_set(2.0)
    np.testing.assert_array_equal(P, render.level0_template_poses(2.0))
    np.testing.assert_array_equal(cli.view_poses(2.0), P)
    path = str(tmp_path / "obj_poses_level0.npy")
    np.save(path, torch.load(os.path.join(golden_dir, "template_poses_level0.pt"))["obj_poses"].numpy())
    P, idx = cli.view_set(400.0, path)
    assert P.shape == (42, 4, 4) and np.array_equal(idx, np.arange(42))
    with pytest.raises(ValueError):
        cli.view_set(400.0, path, 1, "all")


def test_ism_cli_view_selection_and_flags():
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, run_sam6d
    d = ism_cli.get_parser().parse_args([])
    assert (d.aggregation_function, d.level_templates, d.pose_distribution) == ("avg_5", 0, "all")
    np.testing.assert_array_equal(ism_cli.ism_views(42), np.arange(42))
    np.testing.assert_array_equal(ism_cli.ism_views(17), np.arange(17))                 # default: every view in the directory
    np.testing.assert_array_equal(ism_cli.ism_views(357, 2, "upper"), render.template_view_set(2, "upper")[1])
    with pytest.raises(ValueError):
        ism_cli.ism_views(42, 2, "all")                                                 # templates rendered with other flags
    req = ["--cad_path", "o.ply", "--rgb_path", "r.png", "--depth_path", "d.png", "--cam_path", "c.json", "--output_dir", "out"]
    a = run_sam6d.get_parser().parse_args(req)
    assert (a.aggregation_function, a.level_templates, a.pose_distribution) == ("avg_5", 0, "all")
    a = run_sam6d.get_parser().parse_args(req + ["--aggregation_function", "median", "--level_templates", "2", "--pose_distribution", "upper"])
    assert (a.aggregation_function, a.level_templates, a.pose_distribution) == ("median", 2, "upper")
    for bad in (["--aggregation_function", "avg_3"], ["--level_templates", "5"], ["--pose_distribution", "side"]):
        with pytest.raises(SystemExit):
            run_sam6d.get_parser().parse_args(req + bad)


def test_sam6d_rejects_unknown_settings_before_building_models():
    from sam6d_b200.pipeline import SAM6D
    for kw in (dict(level_templates=3), dict(pose_distribution="lower"), dict(aggregation_function="avg_3")):
        with pytest.raises(ValueError):
            SAM6D(**kw)
