"""CPU: ISM references from a BOP PBR split (sam6d_b200/pbr.py) against the reference's own BOPTemplatePBR on the synthetic split
of tests/golden/ism_pbr.pt (tools/make_golden_ism_pbr.py): scan order and its max_num_frames quirk, the shuffle (against pandas
too), the strict visibility filter, the selection at level 0 and 1, the composite and crops of the numpy oracle the GPU test
holds the kernel to, and the argument errors of SAM6D and run_sam6d."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _pbr_oracle as po   # noqa: E402


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ism_pbr.pt"), weights_only=False)


@pytest.fixture(scope="module")
def root(gold, tmp_path_factory):
    return po.write_split(gold["files"], str(tmp_path_factory.mktemp("bop")))


def _keys(rows, index=None):
    index = range(len(rows)) if index is None else index
    return [(str(rows.scene_id[i]), int(rows.frame_id[i]), int(rows.idx_obj[i])) for i in index]


def test_scan_order_and_max_num_frames(gold, root):
    from sam6d_b200 import pbr
    rows = pbr.scan_rows(root, max_num_frames=gold["max_num_frames"])
    g = gold["levels"][0]
    assert _keys(rows) == [tuple(k) for k in g["raw_keys"]]
    assert np.array_equal(rows.visib_fract, g["raw_visib"])
    # the first scene has 8 frames: the break after the rows of position max_num_frames + 1 keeps max_num_frames + 2 of them
    assert sorted(set(int(f) for s, f in zip(rows.scene_id, rows.frame_id) if s == "000000")) == [0, 1, 2, 3, 5, 6]
    assert "models" not in set(rows.scene_id)
    assert len(pbr.scan_rows(root)) > len(rows)                   # max_num_frames defaults to 1000
    assert set(pbr.scan_rows(root, max_num_scenes=1).scene_id) == {"000000"}
    for i in range(len(rows)):                                    # poses: cam_R_m2c, cam_t_m2c (mm)
        assert rows.poses[i, 3].tolist() == [0, 0, 0, 1] and abs(np.linalg.det(rows.poses[i, :3, :3]) - 1) < 1e-9


@pytest.mark.parametrize("n", [0, 1, 2, 7, 39, 1000])
def test_shuffle_matches_pandas(n):
    import pandas as pd
    from sam6d_b200 import pbr
    df = pd.DataFrame({"a": np.arange(n)})
    assert np.array_equal(df.sample(frac=1, random_state=2021).index.to_numpy(), pbr.shuffle_order(n))


def test_shuffle_and_filter_match_golden(gold, root):
    from sam6d_b200 import pbr
    raw = pbr.scan_rows(root, max_num_frames=gold["max_num_frames"])
    shuffled = raw.take(pbr.shuffle_order(len(raw)))
    assert _keys(shuffled) == [tuple(k) for k in gold["levels"][0]["shuffled_keys"]]
    rows = pbr.scan_split(root, max_num_frames=gold["max_num_frames"])
    at = shuffled.visib_fract == 0.8
    assert at.any(), "the split should hold visib_fract values of exactly 0.8"
    assert _keys(rows) == [k for k, v in zip(_keys(shuffled), shuffled.visib_fract) if v > 0.8]
    assert 9 not in set(rows.obj_id.tolist())


@pytest.mark.parametrize("level", [0, 1])
def test_selection_matches_golden(gold, root, level):
    """with the reference's view set in its order the selection is the reference's; with the project's view set (the same
    views, ordered by elevation and azimuth) it is the reference's in that order"""
    from sam6d_b200 import pbr, render
    g = gold["levels"][level]
    rows = pbr.scan_split(root, max_num_frames=gold["max_num_frames"])
    want = [[tuple(k) for k in obj] for obj in g["selected"]]
    sel = pbr.select_references(rows, gold["obj_ids"], g["template_poses"], np.random.RandomState(g["np_seed"]))
    assert [_keys(rows, s) for s in sel] == want
    np.random.seed(g["np_seed"])                                   # the default RNG is numpy's global one
    assert np.array_equal(pbr.select_references(rows, gold["obj_ids"], g["template_poses"]), sel)
    union, index = render.template_view_set(level, "all")
    ours = union[index]
    d = np.linalg.norm(ours[:, None, 2, :3] - g["template_poses"][None, :, 2, :3], axis=-1)
    perm = d.argmin(axis=1)
    assert d.min(axis=1).max() < 1e-4 and len(set(perm.tolist())) == len(ours)     # its files hold the views to ~1e-5
    sel2 = pbr.select_references(rows, gold["obj_ids"], ours, np.random.RandomState(g["np_seed"]))
    assert [_keys(rows, s) for s in sel2] == [[obj[p] for p in perm] for obj in want]


def test_no_rows_for_an_object(gold, root):
    from sam6d_b200 import pbr
    rows = pbr.scan_split(root)
    with pytest.raises(ValueError, match="object 9"):
        pbr.select_references(rows, [1, 9], gold["levels"][0]["template_poses"], np.random.RandomState(0))


def test_composite_matches_pil():
    """every (pixel value, mask value) pair, through PIL's Image.composite and the reference's / 255 -> float32"""
    from PIL import Image
    v = np.arange(256, dtype=np.uint8)
    rgb = np.stack([np.repeat(v[:, None], 256, 1), np.repeat(v[::-1, None], 256, 1), np.repeat(v[:, None], 256, 1)], axis=-1)
    mask = np.repeat(v[None, :], 256, 0)
    pil = np.array(Image.composite(Image.fromarray(rgb), Image.new("RGB", (256, 256), (0, 0, 0)), Image.fromarray(mask)))
    assert np.array_equal(po.composite(rgb, mask), pil)
    assert po.getbbox(mask) == Image.fromarray(mask).getbbox()
    assert po.getbbox(np.zeros((4, 5), np.uint8)) is None and Image.fromarray(np.zeros((4, 5), np.uint8)).getbbox() is None


def test_oracle_crops_match_golden(gold, root):
    from sam6d_b200 import pbr
    rows = pbr.scan_rows(root)
    where = {k: i for i, k in enumerate(_keys(rows))}
    crops = gold["levels"][0]["crops"]
    assert len(crops) >= 4
    for c in crops:
        i = where[tuple(c["key"])]
        _, rgb, m = po.reference_crop(pbr.decode_rgb(rows.rgb_path[i]), pbr.decode_mask(rows.mask_path(i)))
        assert torch.equal(rgb, po.unpack(c["templates"])), c["key"]
        assert torch.equal(m, po.unpack(c["template_masks"])), c["key"]


def _no_models(monkeypatch):
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli

    def refuse(*a, **k):
        raise AssertionError("a model was built")
    monkeypatch.setattr(ism_cli, "build_models", refuse)
    monkeypatch.setattr(pem_cli, "build_model", refuse)


def test_sam6d_argument_errors(root, monkeypatch):
    from sam6d_b200.pipeline import SAM6D
    _no_models(monkeypatch)
    with pytest.raises(ValueError, match="pbr_root"):
        SAM6D(rendering_type="pbr", device="cpu")
    with pytest.raises(NotImplementedError, match="all"):
        SAM6D(rendering_type="pbr", pbr_root=root, pose_distribution="upper", device="cpu")
    with pytest.raises(FileNotFoundError):
        SAM6D(rendering_type="pbr", pbr_root=os.path.join(root, "nowhere"), device="cpu")
    with pytest.raises(ValueError, match="rendering_type"):
        SAM6D(rendering_type="blender", device="cpu")


def test_onboard_needs_obj_ids(root, monkeypatch):
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli
    from sam6d_b200.pipeline import SAM6D
    monkeypatch.setattr(ism_cli, "build_models", lambda *a, **k: (None, None))
    monkeypatch.setattr(pem_cli, "build_model", lambda *a, **k: None)
    m = SAM6D(rendering_type="pbr", pbr_root=root, device="cpu")
    with pytest.raises(ValueError, match="obj_id"):
        m.onboard("never_read.ply")
    with pytest.raises(ValueError, match="obj_ids"):
        m.onboard_objects(["a.ply", "b.ply"])
    assert m._pbr_rows is None                                      # nothing scanned yet


def test_run_sam6d_flags(root, monkeypatch):
    from sam6d_b200.cli import run_sam6d
    _no_models(monkeypatch)
    a = run_sam6d.get_parser().parse_args(["--output_dir", "o", "--cad_path", "c.ply", "--rgb_path", "r", "--depth_path", "d", "--cam_path", "k"])
    assert (a.rendering_type, a.pbr_root, a.pbr_split) == ("pyrender", None, "train_pbr")
    base = ["--output_dir", "o", "--cad_path", "c.ply", "--rgb_path", "r", "--depth_path", "d", "--cam_path", "k", "--rendering_type", "pbr"]
    with pytest.raises(SystemExit):
        run_sam6d.main(base + ["--pbr_root", root])                   # no --obj_ids
    with pytest.raises(SystemExit):
        run_sam6d.main(base + ["--obj_ids", "1"])                     # no --pbr_root
    with pytest.raises(SystemExit):
        run_sam6d.get_parser().parse_args(base[:-1] + ["blender"])
    a = run_sam6d.get_parser().parse_args(base + ["--pbr_root", root, "--pbr_split", "s", "--obj_ids", "1", "5"])
    assert (a.rendering_type, a.pbr_root, a.pbr_split, a.obj_ids) == ("pbr", root, "s", [1, 5])
