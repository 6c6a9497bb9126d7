"""CPU: the host side of SAM-6D over a BOP test split (sam6d_b200/bop.py, cli/run_bop.py) against tests/golden/bop_test.pt,
which holds a synthetic split and what the reference's own BOPTestset, test_bop.py and Detections.save_to_file made of it
(tools/make_golden_bop_test.py)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from sam6d_b200 import bop

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bop_golden as bg   # noqa: E402


@pytest.fixture(scope="module")
def gold(golden_dir):
    return bg.load(golden_dir)


@pytest.fixture(scope="module")
def split(gold, tmp_path_factory):
    return bg.write_split(gold, tmp_path_factory.mktemp("bop"))


def test_split_names():
    assert bop.split_name("tless") == bop.split_name("hb") == "test_primesense"
    assert [bop.split_name(d) for d in ("ycbv", "lmo", "tudl", "icbin", "itodd")] == ["test"] * 5
    assert bop.model_dir("tless") == "models_cad" and bop.model_dir("ycbv") == "models"


def test_scan_test_split(split):
    frames = bop.scan_test_split(split, "lmo")
    assert [(f.scene_id, f.frame_id) for f in frames] == [(2, 3), (7, 1), (7, 2), (9, 4)]
    exts = [os.path.relpath(f.rgb_path, split) for f in frames]
    assert exts[0] == "lmo/test/000002/rgb/000003.png" and exts[1] == "lmo/test/000007/rgb/000001.jpg"
    assert exts[3] == "lmo/test/000009/gray/000004.tif"
    assert all(f.depth_path == os.path.join(split, "lmo", "test", f"{f.scene_id:06d}", "depth", f"{f.frame_id:06d}.png") for f in frames)
    assert [f.depth_scale for f in frames] == [0.1, 1.0, 1.0, 0.1] and len(frames[0].cam_K) == 9
    # the PEM's reads of the same images
    for f in frames:
        assert bop.frame_paths(split, "lmo", f.scene_id, f.frame_id) == (f.rgb_path, f.depth_path, f.cam_K, f.depth_scale)
    gray = bop.decode_rgb(frames[3].rgb_path)
    assert gray.shape == (48, 64, 3) and (gray[..., 0] == gray[..., 1]).all() and (gray[..., 0] == gray[..., 2]).all()


def test_primesense_and_gray_depth(tmp_path):
    """tless reads test_primesense; a gray scene without depth/<id>.png takes the image path with gray replaced by depth"""
    from PIL import Image
    scene = tmp_path / "tless" / "test_primesense" / "000001"
    (scene / "gray").mkdir(parents=True)
    (scene / "depth").mkdir()
    Image.fromarray(np.zeros((4, 6), np.uint8)).save(scene / "gray" / "000007.tif")
    (scene / "scene_camera.json").write_text(json.dumps({"7": {"cam_K": list(range(9)), "depth_scale": 0.5}}))
    (tmp_path / "tless" / "test" / "000001").mkdir(parents=True)          # the other split is not read
    frames = bop.scan_test_split(str(tmp_path), "tless")
    assert len(frames) == 1 and frames[0].depth_path == str(scene / "depth" / "000007.tif") and frames[0].depth_scale == 0.5
    with pytest.raises(FileNotFoundError):
        bop.scan_test_split(str(tmp_path), "ycbv")


def test_objects_and_template_views(split, tmp_path):
    objs = bop.load_objects(split, "lmo")
    assert objs.ids == [1, 5] and np.array_equal(objs.diameters, [120.0 / 1000.0, 90.0 / 1000.0])
    assert objs.index(5) == 1
    with pytest.raises(ValueError):
        objs.index(3)
    assert bop.template_views(42) == list(range(42))
    assert bop.template_views(162) == [int(162 / 42 * v) for v in range(42)] and bop.template_views(162)[1] == 3
    rgbs, masks, xyzs = bop.load_templates(os.path.join(split, "BOP-Templates"), "lmo", 5)
    assert len(rgbs) == 42 and rgbs[0].shape == (32, 32, 3) and masks[0].dtype == np.uint8 and xyzs[0].dtype == np.float32
    (tmp_path / "tless" / "models_cad").mkdir(parents=True)
    (tmp_path / "tless" / "models_cad" / "obj_000003.ply").write_text("")
    (tmp_path / "tless" / "models_cad" / "models_info.json").write_text(json.dumps({"3": {"diameter": 50.0}}))
    t = bop.load_objects(str(tmp_path), "tless")
    assert t.ids == [3] and t.diameters[0] == 0.05


def test_category_ids_against_reference(gold):
    """Detections.save_to_file + convert_npz_to_json: index + 1, and lmo_object_ids[index] on lmo"""
    from sam6d_b200.pipeline import ism_records
    assert bop.category_ids("lmo", 8) == [1, 5, 6, 8, 9, 10, 11, 12]
    assert bop.category_ids("ycbv", 3) == [1, 2, 3]
    with pytest.raises(ValueError):
        bop.category_ids("lmo", 9)
    g = gold["ism"]
    for name, ref in g["records"].items():
        cats = np.asarray(bop.category_ids(name, 8))[g["object_ids"].numpy()]
        counts = [r["segmentation"]["counts"] for r in ref]
        ours = ism_records(g["boxes"].numpy(), g["scores"].numpy(), counts, g["masks"]["shape"][1:], g["runtime"], category_ids=cats)
        for r in ours:
            r.update(scene_id=48, image_id=3)
        assert ours == ref, name
        assert [list(r) for r in ours] == [list(r) for r in ref]                 # key order of the JSON


def test_grouping_and_score_filter(gold):
    groups = bop.group_detections(gold["detections"])
    keys = [f"{s:06d}_{i:06d}" for (s, i), _ in groups]
    assert keys == [im["key"] for im in gold["images"]]
    for (_, dets), im in zip(groups, gold["images"]):
        kept = [d for d in dets if d["score"] > bop.SEG_FILTER_SCORE]
        if im["empty"]:
            assert all(d["score"] <= 0.25 for d in dets)
            continue
        assert im["n_dets"] == len(dets)
        assert set(im["score"]) <= {float(np.float32(d["score"])) for d in kept} and len(kept) > len(im["score"])
        assert any(d["score"] == 0.25 for d in dets)                          # 0.25 itself is dropped (strict >)


def test_csv_rows_against_reference(gold):
    """test_bop.py's lines from the stub Net's outputs: every field but the time equal as text"""
    so, bs = gold["stub_out"], gold["stub_bs"]
    lines, pos = [], 0
    for im in gold["images"]:
        if im["empty"]:
            continue
        n = len(im["obj_id"])
        sl = slice(pos, pos + n)
        pos += n
        scores = (so["pred_pose_score"][sl] * torch.tensor(im["score"], dtype=torch.float32)).numpy()
        R, t = so["pred_R"][sl].reshape(-1, 9).numpy(), so["pred_t"][sl].numpy() * 1000
        s, i = (int(x) for x in im["key"].split("_"))
        lines += bop.csv_rows(s, i, im["obj_id"], scores, R, t, im["seg_time"])
    ref = gold["csv_lines"]
    assert len(lines) == len(ref) == pos and bs < max(len(im.get("obj_id", [])) for im in gold["images"])
    for a, b in zip(lines, ref):
        assert a.split(",")[:6] == b.split(",")[:6]
        assert a.endswith("\n") and float(b.split(",")[6]) >= float(a.split(",")[6])


def test_round_trip_table_all_entries():
    """the 768 entries against a literal restatement in numpy float32, and against torchvision's transforms on an image"""
    table = bop.round_trip_table()
    f = np.float32
    for c, (m, s) in enumerate(zip((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))):
        for v in range(256):
            x = f(v) / f(255)
            y = (x - f(m)) / f(s)
            z = (y - f(-m / s)) / f(1 / s)
            assert table[c, v] == np.uint8(np.clip(z, f(0), f(1)) * f(255)), (c, v)
    assert (table != np.arange(256)[None]).any()                            # the round trip is not the identity
    import torchvision.transforms as T
    from PIL import Image
    img = np.stack([np.arange(256, dtype=np.uint8).reshape(16, 16)] * 3, axis=-1)
    img[..., 1] = img[..., 1][::-1]
    fwd = T.Compose([T.ToTensor(), T.Normalize(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))])
    inv = T.Normalize(mean=[-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225], std=[1 / 0.229, 1 / 0.224, 1 / 0.225])
    ref = np.uint8(inv(fwd(Image.fromarray(img))).numpy().transpose(1, 2, 0).clip(0, 1) * 255)
    assert np.array_equal(bop.round_trip(img), ref)


def test_pem_rand_chunks():
    """one torch.rand(chunk, n) per chunk of 16 instances from one generator that continues across images"""
    g = torch.Generator().manual_seed(1)
    a = bop.pem_rand(g, 37, 12, "cpu")
    b = bop.pem_rand(g, 3, 12, "cpu")
    h = torch.Generator().manual_seed(1)
    ref = [torch.rand(16, 12, generator=h), torch.rand(16, 12, generator=h), torch.rand(5, 12, generator=h), torch.rand(3, 12, generator=h)]
    assert torch.equal(a, torch.cat(ref[:3])) and torch.equal(b, ref[3])
    assert bop.pem_rand(g, 0, 12, "cpu").shape == (0, 12)


def test_pem_depth_formula():
    raw = np.arange(0, 65536, 7, dtype=np.uint16)
    d = bop.pem_depth(raw, 0.1)
    assert d.dtype == np.float32 and np.array_equal(d, (raw / 1000.0 * 0.1).astype(np.float32))
    custom = raw.astype(np.float32) * 0.1 / 1000.0
    assert (d != custom).any()


def test_cli_argument_errors(tmp_path):
    from sam6d_b200.cli import run_bop
    (tmp_path / "ycbv").mkdir()
    base = ["--bop_root", str(tmp_path), "--dataset_name", "ycbv", "--output_dir", str(tmp_path / "out")]
    for extra in (["--stage", "pem"],                                           # no --template_dir
                  ["--template_dir", "t", "--detections", "d.json"],           # --detections with both
                  ["--template_dir", "t", "--stage", "pem", "--detections", str(tmp_path / "missing.json")],
                  ["--stage", "ism", "--max_frames", "0"],
                  ["--stage", "nope"]):
        with pytest.raises(SystemExit):
            run_bop.main(base + extra)
    with pytest.raises(SystemExit):
        run_bop.main(["--bop_root", str(tmp_path), "--dataset_name", "lmo", "--output_dir", "o", "--stage", "ism"])
    args = run_bop.get_parser().parse_args(base + ["--template_dir", "t", "--rendering_type", "pbr", "--segmentor_model", "fastsam",
                                                   "--fastsam_model", "FastSAM-s", "--level_templates", "1", "--aggregation_function", "median"])
    assert args.stage == "both" and args.rendering_type == "pbr" and args.level_templates == 1 and args.fastsam_model == "FastSAM-s"
