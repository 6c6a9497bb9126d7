"""GPU: SAM-6D over a BOP test split (SAM6D.run_bop_ism / run_bop_pem, cli/run_bop.py).

- bop.pem_instances against the reference's BOPTestset.__getitem__ (tests/golden/bop_test.pt), bit for bit at its sample
  indices; the custom path's float32 depth formula gives other points.
- run_bop_ism on a split made of the example frame: each frame's records are detect_objects' on the round-tripped image, with
  the BOP ids filled in, and their RLE decodes to the device masks.
- run_bop_pem: its rows are Net.forward on the instances, one instance at a time, with test_bop.py's chunked uniforms; the
  image whose detections are all dropped is skipped.
- run_bop --stage both writes the JSON and the CSV."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from sam6d_b200 import bop

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bop_golden as bg   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold(golden_dir):
    return bg.load(golden_dir)


@pytest.fixture(scope="module")
def lmo_split(gold, tmp_path_factory):
    return bg.write_split(gold, tmp_path_factory.mktemp("bop"))


def _image_inputs(root, key):
    s, i = (int(x) for x in key.split("_"))
    rgb_path, depth_path, K, scale = bop.frame_paths(root, "lmo", s, i)
    return bop.decode_pem_image(rgb_path), bop.decode_depth(depth_path), K, scale


def test_instances_match_reference(gold, lmo_split, monkeypatch):
    objs = bop.load_objects(lmo_split, "lmo")
    mp = np.stack([bg.unpack(gold["model_points"][o]).numpy() for o in objs.ids])
    groups = dict(((f"{s:06d}_{i:06d}", d) for (s, i), d in bop.group_detections(gold["detections"])))
    n_inst = 0
    for im in gold["images"]:
        image, raw, K, scale = _image_inputs(lmo_split, im["key"])
        ref = bg.instance(im) if not im["empty"] else None
        ci = ref["choose_idx"] if ref is not None else np.zeros((0, 2048), np.int64)
        data, kept, _ = bop.pem_instances(groups[im["key"]], image, raw, K, scale, objs, mp, choose_idx=ci)
        if im["empty"]:
            assert not kept and data["pts"].shape[0] == 0
            continue
        n_inst += len(kept)
        assert torch.equal(data["pts"].cpu(), ref["pts"]), im["key"]
        assert torch.equal(data["rgb"].cpu(), ref["rgb"]), im["key"]
        assert torch.equal(data["rgb_choose"].cpu(), ref["rgb_choose"]), im["key"]
        assert torch.equal(data["model"].cpu(), torch.from_numpy(mp)[ref["obj"]]), im["key"]     # BOPTestset's model rows
        assert torch.equal(data["obj"].cpu(), ref["obj"]) and torch.equal(data["score"].cpu(), ref["score"])
        assert [d["category_id"] for d in kept] == im["obj_id"]
    assert n_inst == 12
    # the custom path's depth (float32 raw * depth_scale / 1000.0) gives other points on at least one instance
    monkeypatch.setattr(bop, "pem_depth", lambda r, s: np.asarray(r).astype(np.float32) * s / 1000.0)
    differ = 0
    for im in gold["images"]:
        if im["empty"]:
            continue
        image, raw, K, scale = _image_inputs(lmo_split, im["key"])
        ref = bg.instance(im)
        data, kept, _ = bop.pem_instances(groups[im["key"]], image, raw, K, scale, objs, mp, choose_idx=ref["choose_idx"])
        differ += len(kept) != len(im["obj_id"]) or not torch.equal(data["pts"].cpu(), ref["pts"])
    assert differ >= 1


_MODEL = {}


def _sam6d():
    from sam6d_b200.pipeline import SAM6D
    if "m" not in _MODEL:
        _MODEL["m"] = SAM6D(segmentor="fastsam", random_weights=True, confidence_thresh=-1, det_score_thresh=-1)
    return _MODEL["m"]


def test_run_bop_pem_matches_forward(gold, lmo_split, tmp_path):
    from sam6d_b200 import meshio
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli
    from sam6d_b200.pipeline import pem_template_bank
    model = _sam6d()
    det_path = tmp_path / "dets.json"
    json.dump(gold["detections"], open(det_path, "w"))
    out = tmp_path / "result_lmo.csv"
    tdir = os.path.join(lmo_split, "BOP-Templates")
    lines = model.run_bop_pem(str(det_path), lmo_split, "lmo", tdir, str(out), rng=np.random.RandomState(3))
    assert open(out).read() == "".join(lines)
    # the same draws by hand, then every instance alone through Net.forward with its row of the chunked uniforms
    rng = np.random.RandomState(3)
    objs = bop.load_objects(lmo_split, "lmo")
    meshes = [meshio.load_ply_mesh(p) for p in objs.ply_paths]
    mp = np.stack([meshio.sample_surface(m.vertices, m.faces, 1024, rng) / 1000.0 for m in meshes]).astype(np.float32)
    banks = [pem_template_bank(model.pem, *bop.load_templates(tdir, "lmo", i), rng=rng, device=model.device) for i in objs.ids]
    g = torch.Generator(device="cuda")
    g.manual_seed(pem_cli.RD_SEED)
    n_rand = model.pem.coarse_point_matching.cfg.nproposal1 * 3
    expect, skipped = [], []
    for (s, i), dets in bop.group_detections(gold["detections"]):
        image, raw, K, scale = _image_inputs(lmo_split, f"{s:06d}_{i:06d}")
        data, kept, _ = bop.pem_instances(dets, image, raw, K, scale, objs, mp, rng=rng)
        if not kept:
            skipped.append((s, i))
            continue
        rand = torch.cat([torch.rand(min(16, len(kept) - c), n_rand, generator=g, device="cuda") for c in range(0, len(kept), 16)])
        for k, o in enumerate(data["obj"].tolist()):
            one = {key: data[key][k:k + 1] for key in ("pts", "rgb", "rgb_choose", "model")}
            one["dense_po"], one["dense_fo"] = banks[o][0].reshape(1, 2048, 3), banks[o][1].reshape(1, 2048, -1)
            with torch.no_grad():
                r = model.pem(one, rand=rand[k:k + 1])
            score = (r["pred_pose_score"] * data["score"][k:k + 1]).cpu().numpy()
            expect += bop.csv_rows(s, i, [kept[k]["category_id"]], score, r["pred_R"].reshape(-1, 9).cpu().numpy(),
                                   r["pred_t"].cpu().numpy() * 1000, 0.0)
    assert skipped == [(7, 2)] and len(lines) == len(expect) == 12
    strip = lambda ls: [x.rsplit(",", 1)[0] for x in ls]                      # noqa: E731
    assert strip(lines) == strip(expect)
    assert all(float(x.rsplit(",", 1)[1]) > 0 for x in lines)


def _ycbv_split(golden_dir, root):
    """the example frame as a BOP split: scene 1 frame 0 (PNG), scene 3 frame 5 (JPEG); two objects, the convex hull of the
    example's model points at two scales, with the PEM's 42 template views rendered from them"""
    import cv2
    from scipy.spatial import ConvexHull
    from sam6d_b200 import meshio
    from sam6d_b200.pipeline import render_templates, template_arrays
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    pts = g["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    faces = np.array([[remap[a] for a in s] for s in hull.simplices], dtype=np.int64)
    cols = np.random.RandomState(0).randint(40, 255, (len(hull.vertices), 3)).astype(np.uint8)
    ds = os.path.join(root, "ycbv")
    os.makedirs(os.path.join(ds, "models"))
    info = {}
    for oid, sc in ((1, 1.0), (2, 0.7)):
        v = (pts[hull.vertices] * sc).astype(np.float32)
        with open(os.path.join(ds, "models", f"obj_{oid:06d}.ply"), "w") as fh:
            fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\n"
                     "property uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                     % (len(v), len(faces)))
            for p, c in zip(v, cols):
                fh.write("%f %f %f %d %d %d\n" % (p[0], p[1], p[2], c[0], c[1], c[2]))
            for f in faces:
                fh.write("3 %d %d %d\n" % tuple(f))
        info[str(oid)] = {"diameter": float(2 * np.linalg.norm(v, axis=1).max())}
        out, _ = render_templates(meshio.Mesh(vertices=v, faces=faces, colors=cols), 192)
        rgbs, masks, xyzs = template_arrays(out)
        tdir = os.path.join(root, "templates", "ycbv", f"obj_{oid:06d}")
        os.makedirs(tdir)
        for k in range(42):
            cv2.imwrite(os.path.join(tdir, f"rgb_{k}.png"), rgbs[k][:, :, ::-1])
            cv2.imwrite(os.path.join(tdir, f"mask_{k}.png"), masks[k])
            np.save(os.path.join(tdir, f"xyz_{k}.npy"), xyzs[k].astype(np.float16))
    json.dump(info, open(os.path.join(ds, "models", "models_info.json"), "w"))
    rgb, depth = g["rgb"].numpy().astype(np.uint8), g["depth"].numpy().astype(np.uint16)
    for scene, fid, ext in ((1, 0, "png"), (3, 5, "jpg")):
        sdir = os.path.join(ds, "test", f"{scene:06d}")
        os.makedirs(os.path.join(sdir, "rgb"))
        os.makedirs(os.path.join(sdir, "depth"))
        cv2.imwrite(os.path.join(sdir, "rgb", f"{fid:06d}.{ext}"), rgb[:, :, ::-1])
        cv2.imwrite(os.path.join(sdir, "depth", f"{fid:06d}.png"), depth)
        json.dump({str(fid): {"cam_K": [float(x) for x in np.asarray(g["cam_K"]).reshape(-1)], "depth_scale": float(g["depth_scale"])}},
                  open(os.path.join(sdir, "scene_camera.json"), "w"))
    return root


@pytest.fixture(scope="module")
def ycbv(golden_dir, tmp_path_factory):
    return _ycbv_split(golden_dir, str(tmp_path_factory.mktemp("ycbv")))


def test_run_bop_ism_matches_detect_objects(ycbv, tmp_path):
    model = _sam6d()
    objects = model.onboard_bop(ycbv, "ycbv", template_size=192, rng=np.random.RandomState(0))
    assert objects.obj_ids == [1, 2]
    out = tmp_path / "result_ycbv.json"
    recs = model.run_bop_ism(ycbv, "ycbv", objects, str(out))
    assert json.load(open(out)) == json.loads(json.dumps(recs))
    frames = bop.scan_test_split(ycbv, "ycbv")
    assert len(frames) == 2
    strip = lambda rs: [{k: v for k, v in r.items() if k not in ("time", "scene_id", "image_id")} for r in rs]   # noqa: E731
    for f in frames:
        rgb = bop.round_trip(bop.decode_rgb(f.rgb_path))
        res = model.detect_objects(rgb, bop.decode_depth(f.depth_path), f.cam_K, f.depth_scale, objects)
        mine = [r for r in recs if (r["scene_id"], r["image_id"]) == (f.scene_id, f.frame_id)]
        assert res.ism and strip(mine) == strip(res.ism)
        assert [r["category_id"] for r in mine] == [[1, 2][o] for o in res.obj.tolist()]
        assert all(0 < r["time"] for r in mine) and len({r["time"] for r in mine}) == 1
        # the RLE of every record decodes to the device mask
        for r, m in zip(mine, res.masks):
            flat = np.zeros(int(np.prod(r["segmentation"]["size"])), np.uint8)
            pos = np.cumsum([0] + r["segmentation"]["counts"])
            for k in range(1, len(pos) - 1, 2):
                flat[pos[k]:pos[k + 1]] = 1
            assert np.array_equal(flat.reshape(r["segmentation"]["size"], order="F"), (m > 0).cpu().numpy().astype(np.uint8))
    print(f"run_bop_ism: {len(recs)} records over {len(frames)} frames")


def test_run_bop_cli_both(ycbv, tmp_path):
    from sam6d_b200.cli import run_bop
    out = tmp_path / "out"
    np.random.seed(0)
    assert run_bop.main(["--bop_root", ycbv, "--dataset_name", "ycbv", "--template_dir", os.path.join(ycbv, "templates"),
                         "--output_dir", str(out), "--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1",
                         "--template_size", "192", "--max_frames", "1"]) == 0
    recs = json.load(open(out / "result_ycbv.json"))
    assert recs and {(r["scene_id"], r["image_id"]) for r in recs} == {(1, 0)}
    assert list(recs[0]) == ["scene_id", "image_id", "category_id", "bbox", "score", "time", "segmentation"]
    rows = open(out / "result_ycbv.csv").read().splitlines()
    kept = [r for r in recs if r["score"] > 0.25]
    print(f"run_bop --stage both: {len(recs)} detections ({len(kept)} above 0.25), {len(rows)} poses")
    for row in rows:
        f = row.split(",")
        assert len(f) == 7 and f[:2] == ["1", "0"] and len(f[4].split(" ")) == 9 and len(f[5].split(" ")) == 3
    assert len(rows) <= len(kept)
